"""Times SORT on the device (gast_b200.tracking) against the reference's per-frame host tracker.

  - DeviceSort.update_chunk on three cases, CUDA events after warm-up: a baseball-shaped chunk (277 frames, 1 - 3
    persons plus clutter), a crowded chunk (277 frames, 30 persons) and 64 baseball-shaped videos in one launch;
  - the numpy restatement of the reference's Sort (tests/sortref.py: scipy-equal assignment in Python, numpy Kalman
    filter; the reference itself uses numba's iou and scipy's solver) per-frame update on the baseball-shaped chunk,
    host clock;
  - video_boxes over a 277-frame 1920 x 1080 clip with a stand-in net (fixed predictions per frame), once with a
    DeviceSort and once with the restated Sort, host clock around work that ends in a copy to the host.

Three alternated rounds; the card's name, power limit and max SM clock are read in the same run.  Prints one JSON
line.  Usage: python tools/track_bench.py [--rounds 3]
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
from gast_b200 import detection as Dt   # noqa: E402
from gast_b200 import tracking as Tk    # noqa: E402
import detectionref as DR               # noqa: E402
import sortref as R                     # noqa: E402

T = 277


def chunk(seeds, persons, alive):
    seqs = [R.random_sequence(T, s, persons, alive) for s in seeds]
    M = max(1, max(len(f) for s in seqs for f in s))
    packed = [R.pack(s, M) for s in seqs]
    b = torch.from_numpy(np.stack([p[0] for p in packed])).cuda()
    n = torch.from_numpy(np.stack([p[1] for p in packed])).cuda()
    return seqs, b, n


def device_ms(b, n, reps=10):
    S = int(b.shape[0])
    trks = [Tk.DeviceSort(S) for _ in range(reps + 1)]
    trks[0].update_chunk(b, n, skip_empty=False)              # warm-up
    torch.cuda.synchronize()
    times = []
    for trk in trks[1:]:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = trk.update_chunk(b, n, skip_empty=False)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    assert not out[2].any().item()
    return float(np.median(times))


def host_ms(frames):
    s = R.Sort()
    t0 = time.perf_counter()
    for f in frames:
        s.update(f)
    return (time.perf_counter() - t0) * 1e3


class Restated:
    def __init__(self):
        self.s = R.Sort()

    def update(self, d):
        return self.s.update(d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    base_seqs, base_b, base_n = chunk([1], 3, 0.6)
    _, crowd_b, crowd_n = chunk([2], 30, 1.0)
    _, many_b, many_n = chunk(list(range(100, 164)), 3, 0.6)
    preds = torch.from_numpy(np.stack([DR.many_candidates(416, k, seed=k) for k in (5, 9, 17)])).cuda()
    frames = torch.from_numpy(DR.synth_frames(T, 1080, 1920, seed=3)).cuda()

    def net(x, cuda):
        return preds[torch.arange(x.shape[0], device=x.device) % preds.shape[0]]

    def vb(tracker):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = Dt.video_boxes(frames, net, tracker, 416)
        return (time.perf_counter() - t0) * 1e3, out

    vb(Tk.DeviceSort())
    vb(Restated())
    res = {k: [] for k in ('baseball_ms', 'crowded_ms', 'videos64_ms', 'host_baseball_ms', 'video_boxes_device_ms',
                           'video_boxes_host_sort_ms')}
    for _ in range(args.rounds):
        res['baseball_ms'].append(device_ms(base_b, base_n))
        res['host_baseball_ms'].append(host_ms(base_seqs[0]))
        res['crowded_ms'].append(device_ms(crowd_b, crowd_n))
        res['videos64_ms'].append(device_ms(many_b, many_n))
        t, a = vb(Tk.DeviceSort())
        res['video_boxes_device_ms'].append(t)
        t, b = vb(Restated())
        res['video_boxes_host_sort_ms'].append(t)
    res = {k: [round(v, 4) for v in vs] for k, vs in res.items()}
    res['gpu'] = smi
    res['persons_per_frame'] = dict(baseball=[int(base_n.min()), int(base_n.max())],
                                    crowded=[int(crowd_n.min()), int(crowd_n.max())])
    res['video_boxes_rows'] = sum(len(o) for o in a if o is not None)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
