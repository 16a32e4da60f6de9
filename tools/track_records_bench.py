"""Times the crop records on the device (gast_b200.keypoints2d.track_records / record_inverse) and the video_keypoints
path they open, against the host path they replace.

  (a) track_records + record_inverse on a baseball-shaped chunk (277 frames of 1920 x 1080, tracks from DeviceSort
      over synthetic detections), for 1 and for 64 sequences in one launch, 1 and 2 persons: CUDA events over many
      calls after warm-up;
  (b) from update_chunk's outputs to the keypoints on the device, with a stand-in HRNet ((n, 3, 384, 288) -> (n, 17,
      96, 72), restated from tests/test_gpu_zz_keypoints2d.py): video_keypoints on the (rows, counts, status) triple
      against host_tracks + video_keypoints' list path, 1 and 2 persons, alternated, host clock to a synchronise.
      Both give the same keypoints bit for bit; the tool checks it.

Three rounds by default; the card's name, power limit and max SM clock are read in the same run.  Prints one JSON
line.  Usage: python tools/track_records_bench.py [--rounds 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, os.path.join(REPO, 'tests'))
from gast_b200 import keypoints2d as K  # noqa: E402
from gast_b200 import tracking as Tk    # noqa: E402
import keypoints2dref as KR             # noqa: E402
import sortref as R                     # noqa: E402

T, W, H = 277, 1920, 1080


class StandInNet(torch.nn.Module):
    """HRNet's shapes, (n, 3, 384, 288) -> (n, 17, 96, 72): a 4 x 4 average pool and a per-joint mix of the planes
    through a sine, seeded"""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        self.register_buffer('w', torch.rand((17, 3), generator=g) * 4 - 2)
        self.register_buffer('b', torch.rand(17, generator=g) * 6)

    def forward(self, x):
        p = torch.nn.functional.avg_pool2d(x, 4)
        return torch.stack([torch.sin(p[:, 0] * self.w[j, 0] + p[:, 1] * self.w[j, 1] + p[:, 2] * self.w[j, 2] +
                                      self.b[j]) for j in range(17)], 1)


def persons(t, k):
    """k persons walking across a 1920 x 1080 frame, in hundredths, with a little jitter"""
    rng = np.random.default_rng(t)
    rows = []
    for i in range(k):
        x1 = 20000 + 45000 * i + 150 * t + int(rng.integers(-200, 201))
        y1 = 30000 + 2000 * i + int(rng.integers(-200, 201))
        rows.append([x1, y1, x1 + 18000 + int(rng.integers(-300, 301)), y1 + 52000 + int(rng.integers(-300, 301))])
    return np.array(rows, np.float32) / np.float32(100)


def tracks(k, S=1):
    """DeviceSort's (rows, counts, status) over S copies of a 277-frame chunk of k persons"""
    boxes, counts = R.pack([persons(t, k) for t in range(T)], 4)
    trk = Tk.DeviceSort(S)
    b = torch.from_numpy(np.broadcast_to(boxes, (S,) + boxes.shape).copy()).cuda()
    n = torch.from_numpy(np.broadcast_to(counts, (S, T)).copy()).cuda()
    out = trk.update_chunk(b, n)
    if S == 1:
        out = (out[0][0], out[1][0], out[2])
    torch.cuda.synchronize()
    return out


def records_ms(triple, num_person, reps=200):
    for _ in range(10):
        rec = K.track_records(*triple, num_person, (W, H))
        K.record_inverse(rec, (72, 96))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        rec = K.track_records(*triple, num_person, (W, H))
        K.record_inverse(rec, (72, 96))
    e1.record()
    e1.synchronize()
    s = rec.summary.cpu().numpy()
    assert not s[:, 2].any()
    return e0.elapsed_time(e1) / reps, int(s[:, 0].sum())


def keypoints_ms(frames, triple, net, num_person, on_device):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    boxes = triple if on_device else Tk.host_tracks(*triple)
    kp, sc = K.video_keypoints(frames, boxes, net, num_person)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, kp, sc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    frames = torch.from_numpy(KR.synth_frames(T, H, W, seed=3)).cuda()
    net = StandInNet().cuda()
    one = {k: tracks(k) for k in (1, 2)}
    many = {k: tracks(k, 64) for k in (1, 2)}
    for k in (1, 2):                                            # warm-up, and the two paths agree
        _, a, b = keypoints_ms(frames, one[k], net, k, True)
        _, c, d = keypoints_ms(frames, one[k], net, k, False)
        assert torch.equal(a, c) and torch.equal(b, d) and a.shape[1] == T
    res = {}
    for _ in range(args.rounds):
        for k in (1, 2):
            for name, tri in (('records_1seq_%dp_ms' % k, one[k]), ('records_64seq_%dp_ms' % k, many[k])):
                ms, n = records_ms(tri, k)
                res.setdefault(name, []).append(ms)
                res['records_%s' % name[8:-3]] = n
            res.setdefault('keypoints_device_%dp_ms' % k, []).append(keypoints_ms(frames, one[k], net, k, True)[0])
            res.setdefault('keypoints_host_%dp_ms' % k, []).append(keypoints_ms(frames, one[k], net, k, False)[0])
    res = {k: [round(v, 4) for v in vs] if isinstance(vs, list) else vs for k, vs in res.items()}
    res['gpu'] = smi
    print(json.dumps(res))


if __name__ == '__main__':
    main()
