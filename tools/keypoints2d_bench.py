"""Times the 2D pose net's crop and decode on a clip shaped like the baseball demo: 277 frames of 1920 x 1080, one and
two persons per frame, 288 x 384 crops, 72 x 96 heatmaps.

  - one gast_b200.keypoints2d.crop_persons call and one decode_heatmaps call over the whole clip (CUDA events);
  - video_keypoints over the clip with a stand-in net (a 4 x 4 average pool and a per-joint sine), host clock around
    work that ends in a device synchronise;
  - when cv2 and torchvision are importable, the reference's per-frame host flow with the same net, restated with
    the reference's libraries: cv2.warpAffine, ToTensor + Normalize, inputs[:, [2, 1, 0]].cuda(), the net,
    .cpu().numpy() and a numpy get_final_preds (argmax, the quarter-pixel shift loop, np.dot per joint).

The device and host flows run alternately, three rounds each; the card's name and power limit are printed with the
numbers.  Prints one JSON line.  Usage: python tools/keypoints2d_bench.py [--frames 277] [--rounds 3]
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
from gast_b200 import keypoints2d as K  # noqa: E402

H, W = 1080, 1920


class StandInNet(torch.nn.Module):
    """(n, 3, 384, 288) -> (n, 17, 96, 72)"""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        self.register_buffer('w', torch.rand((17, 3), generator=g) * 4 - 2)
        self.register_buffer('b', torch.rand(17, generator=g) * 6)

    def forward(self, x):
        p = torch.nn.functional.avg_pool2d(x, 4)
        return torch.sin(torch.einsum('ncyx,jc->njyx', p, self.w) + self.b[None, :, None, None])


def clip_boxes(T, persons, seed=0):
    """per frame, the tracker's rows (persons, 5): two people walking across the frame"""
    rs = np.random.default_rng(seed)
    out = []
    for t in range(T):
        rows = []
        for p in range(persons):
            x1 = 300 + 800 * p + 2.0 * t + rs.uniform(-5, 5)
            y1 = 200 + rs.uniform(-5, 5)
            rows.append([x1, y1, x1 + 260 + rs.uniform(-10, 10), y1 + 700 + rs.uniform(-10, 10), p + 1])
        out.append(np.array(rows))
    return out


def events_ms(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def host_flow(frames_np, boxes, net, persons, cv2, transforms):
    """the reference's per-frame PreProcess + net + .cpu().numpy() + get_final_preds, restated with its libraries"""
    tf = transforms.Compose([transforms.ToTensor(),
                             transforms.Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225])])
    out = []
    for t in range(len(frames_np)):
        rows = K.select_tracks(boxes[t], persons)
        cs = [K.center_scale(b, H, W) for b in rows[:persons]]
        inputs = torch.cat([tf(cv2.warpAffine(frames_np[t], K.affine_pair(c, s)[0], K.IMAGE_SIZE,
                                              flags=cv2.INTER_LINEAR)).unsqueeze(0) for c, s in cs])
        with torch.no_grad():
            hm = net(inputs[:, [2, 1, 0]].cuda()).cpu().numpy()
        n, J, hh, hw = hm.shape
        flat = hm.reshape(n, J, -1)
        idx, mv = np.argmax(flat, 2), np.amax(flat, 2)
        coords = np.stack([idx % hw, np.floor(idx / hw)], -1).astype(np.float32) * (mv > 0)[..., None]
        for i in range(n):
            for j in range(J):
                px, py = int(math.floor(coords[i, j, 0] + 0.5)), int(math.floor(coords[i, j, 1] + 0.5))
                if 1 < px < hw - 1 and 1 < py < hh - 1:
                    d = np.array([hm[i, j, py, px + 1] - hm[i, j, py, px - 1], hm[i, j, py + 1, px] - hm[i, j, py - 1, px]])
                    coords[i, j] += np.sign(d) * .25
        preds = np.zeros_like(coords)
        for i, (c, s) in enumerate(cs):
            inv = K.inverse_matrix(c, s, (hw, hh))
            for j in range(J):
                preds[i, j] = np.dot(inv, np.array([coords[i, j, 0], coords[i, j, 1], 1.]))[:2]
        out.append(preds)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=277)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('keypoints2d_bench: no CUDA device')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    try:
        import cv2
        import torchvision.transforms as transforms
    except ImportError:
        cv2 = transforms = None
    T = args.frames
    g = torch.Generator(device='cuda').manual_seed(1)
    frames = torch.randint(0, 256, (T, H, W, 3), dtype=torch.uint8, device='cuda', generator=g)
    frames_np = frames.cpu().numpy() if cv2 is not None else None
    net = StandInNet().cuda()
    res = {'gpu': smi, 'frames': T}
    for persons in (1, 2):
        boxes = clip_boxes(T, persons)
        fi, fwd, inv = [], [], []
        for t in range(T):
            for b in K.select_tracks(boxes[t], persons):
                c, s = K.center_scale(b, H, W)
                fi.append(t)
                fwd.append(K.affine_pair(c, s)[0])
                inv.append(K.inverse_matrix(c, s, (72, 96)))
        fi_d = torch.tensor(fi, dtype=torch.int32, device='cuda')
        fwd_d = torch.tensor(np.stack(fwd), device='cuda')
        inv_d = torch.tensor(np.stack(inv), device='cuda')
        hm = torch.rand((len(fi), 17, 96, 72), device='cuda', generator=g)
        crop_ms, dec_ms, vk_s, host_s = [], [], [], []
        for _ in range(args.rounds):
            crop_ms.append(events_ms(lambda: K.crop_persons(frames, fi_d, fwd_d)))
            dec_ms.append(events_ms(lambda: K.decode_heatmaps(hm, inv_d)))
            K.video_keypoints(frames, boxes, net, persons)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            K.video_keypoints(frames, boxes, net, persons)
            torch.cuda.synchronize()
            vk_s.append(time.perf_counter() - t0)
            if cv2 is not None:
                t0 = time.perf_counter()
                host_flow(frames_np, boxes, net, persons, cv2, transforms)
                host_s.append(time.perf_counter() - t0)
        n = len(fi)
        r = {'crops': n, 'crop_ms': [min(crop_ms), max(crop_ms)], 'decode_ms': [min(dec_ms), max(dec_ms)],
             'crop_GBps': [3 * 384 * 288 * 4 * n / max(crop_ms) / 1e6, 3 * 384 * 288 * 4 * n / min(crop_ms) / 1e6],
             'video_keypoints_s': [min(vk_s), max(vk_s)]}
        r['reference_host_flow_s'] = [min(host_s), max(host_s)] if host_s else 'not measured: no cv2/torchvision'
        res['persons_%d' % persons] = r
    print(json.dumps(res))


if __name__ == '__main__':
    main()
