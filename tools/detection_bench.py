"""Times the person detector's letterbox and post-processing on a clip shaped like the baseball demo: 277 frames of
1920 x 1080 at inp_dim 416 (10,647 predictions per frame).

  - one gast_b200.detection.letterbox call and one person_boxes call over the whole clip (CUDA events over many
    calls), with the bytes each kernel must move and the rate that gives;
  - person_boxes on synthetic predictions with 5 - 50 person candidates per frame (two dominant), and a worst case in
    which every row passes the confidence filter;
  - video_boxes over the clip with a stand-in net (fixed predictions) and a stub tracker, host clock around work that
    ends in a device synchronise;
  - when cv2 is importable, the reference's per-frame flow restated with its own libraries: letterbox_image's
    cv2.resize, the upload, write_results' torch loop on the device (mask, corners, max, nonzero, unique, sort and the
    greedy NMS loop), the rescale and clamp loop and one .cpu() per box.

The device and host flows run alternately, three rounds each; the card's name, power limit and max SM clock are
printed with the numbers.  Prints one JSON line.  Usage: python tools/detection_bench.py [--frames 277] [--rounds 3]
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
from gast_b200 import detection as Dt  # noqa: E402
import detectionref as R               # noqa: E402

H, W, D = 1080, 1920, 416


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


def clip_predictions(T):
    """(T, N, 85) float32: per frame 5 - 50 person candidates, two of them dominant"""
    return np.stack([R.many_candidates(D, 5 + (t * 7) % 46, seed=t) for t in range(T)])


def worst_predictions(T):
    """every row passes the 0.7 threshold and is a person"""
    p = R.background(D, 3)
    p[:, 4] = 0.75 + 0.2 * R.uniform(5, p.shape[0])
    p[:, 5] = 0.9
    return np.repeat(p[None], T, 0)


class StandIn:
    def __init__(self, pred):
        self.pred = pred

    def __call__(self, x, cuda):
        return self.pred[:x.shape[0]]


class StubTracker:
    def update(self, dets):
        return np.concatenate([dets, np.arange(1, len(dets) + 1)[:, None]], 1)


def _iou(b1, b2):
    ix1, iy1 = torch.max(b1[:, 0], b2[:, 0]), torch.max(b1[:, 1], b2[:, 1])
    ix2, iy2 = torch.min(b1[:, 2], b2[:, 2]), torch.min(b1[:, 3], b2[:, 3])
    z = torch.zeros(ix2.shape, device=b1.device)
    inter = torch.max(ix2 - ix1 + 1, z) * torch.max(iy2 - iy1 + 1, z)
    a1 = (b1[:, 2] - b1[:, 0] + 1) * (b1[:, 3] - b1[:, 1] + 1)
    a2 = (b2[:, 2] - b2[:, 0] + 1) * (b2[:, 3] - b2[:, 1] + 1)
    return inter / (a1 + a2 - inter)


def reference_flow(frames_np, pred, cv2, conf=0.7, nms=0.4):
    """the reference's per-frame letterbox, write_results(det_hm=True) and rescale, with its own libraries"""
    out = []
    for t in range(len(frames_np)):
        img = frames_np[t]
        h, w = img.shape[:2]
        nw, nh = int(w * min(D / w, D / h)), int(h * min(D / w, D / h))
        canvas = np.full((D, D, 3), 128)
        canvas[(D - nh) // 2:(D - nh) // 2 + nh, (D - nw) // 2:(D - nw) // 2 + nw] = \
            cv2.resize(img, (nw, nh), interpolation=cv2.INTER_CUBIC)
        x = torch.from_numpy(canvas[:, :, ::-1].transpose(2, 0, 1).copy()).float().div(255.0)[None].cuda()
        p = pred[t:t + 1] + x.mean() * 0                     # the net's output, after the upload
        p = p * (p[:, :, 4] > conf).float().unsqueeze(2)
        box = p.new(p.shape)
        box[:, :, 0], box[:, :, 1] = p[:, :, 0] - p[:, :, 2] / 2, p[:, :, 1] - p[:, :, 3] / 2
        box[:, :, 2], box[:, :, 3] = p[:, :, 0] + p[:, :, 2] / 2, p[:, :, 1] + p[:, :, 3] / 2
        p[:, :, :4] = box[:, :, :4]
        ip = p[0]
        mc, mi = torch.max(ip[:, 5:85], 1)
        ip = torch.cat((ip[:, :5], mc.float().unsqueeze(1), mi.float().unsqueeze(1)), 1)
        ip = ip[torch.nonzero(ip[:, 4]).squeeze(), :].view(-1, 7)
        ip = ip[torch.nonzero((ip[:, -1] == 0).float()).squeeze()].view(-1, 7)
        if ip.shape[0] == 0:
            out.append(None)
            continue
        torch.unique(ip[:, -1], sorted=True)
        ip = ip[torch.nonzero(ip[:, -2]).squeeze()].view(-1, 7)
        ip = ip[torch.sort(ip[:, 4], descending=True)[1]]
        for i in range(ip.size(0)):
            if i + 1 > ip.size(0):
                break
            ious = _iou(ip[i].unsqueeze(0), ip[i + 1:])
            ip[i + 1:] *= (ious < nms).float().unsqueeze(1)
            ip = ip[torch.nonzero(ip[:, 4]).squeeze()].view(-1, 7)
        dim = torch.FloatTensor([w, h]).repeat(1, 2).cuda().repeat(ip.size(0), 1)
        sf = torch.min(D / dim, 1)[0].view(-1, 1)
        ip[:, [0, 2]] -= (D - sf * dim[:, 0].view(-1, 1)) / 2
        ip[:, [1, 3]] -= (D - sf * dim[:, 1].view(-1, 1)) / 2
        ip[:, 0:4] /= sf
        for i in range(ip.shape[0]):
            ip[i, [0, 2]] = torch.clamp(ip[i, [0, 2]], 0.0, dim[i, 0])
            ip[i, [1, 3]] = torch.clamp(ip[i, [1, 3]], 0.0, dim[i, 1])
        out.append(np.array([[round(v, 2) for v in list(ip[i, 0:4].cpu().numpy())] for i in range(ip.shape[0])]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=277)
    ap.add_argument('--rounds', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('detection_bench: no CUDA device')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    try:
        import cv2
        cv2.ipp.setUseIPP(False)
    except ImportError:
        cv2 = None
    T = args.frames
    N = R.num_predictions(D)
    g = torch.Generator(device='cuda').manual_seed(1)
    frames = torch.randint(0, 256, (T, H, W, 3), dtype=torch.uint8, device='cuda', generator=g)
    frames_np = frames.cpu().numpy()
    pred = torch.from_numpy(clip_predictions(T)).cuda()
    worst = torch.from_numpy(worst_predictions(T)).cuda()
    sizes = torch.tensor([[W, H]] * T, dtype=torch.int32, device='cuda')
    nw, nh = Dt.letterbox_geometry(W, H, D)
    # bytes each kernel must move: the frames' rows the resize reads and the planes it writes; the objectness sector
    # of every prediction row, the whole row of each candidate, and the outputs
    lb_bytes = T * (min(H, 4 * nh) * W * 3 + 3 * D * D * 4)
    lb_ms, pb_ms, wc_ms, vb_s, ref_s = [], [], [], [], []
    net = StandIn(pred)
    cands = int(sum(5 + (t * 7) % 46 for t in range(T)))
    for _ in range(args.rounds):
        lb_ms.append(events_ms(lambda: Dt.letterbox(frames, D)))
        pb_ms.append(events_ms(lambda: Dt.person_boxes(pred, sizes, D)))
        wc_ms.append(events_ms(lambda: Dt.person_boxes(worst, sizes, D), reps=3))
        Dt.video_boxes(frames, net, StubTracker(), D)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        Dt.video_boxes(frames, net, StubTracker(), D)
        torch.cuda.synchronize()
        vb_s.append(time.perf_counter() - t0)
        if cv2 is not None:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            reference_flow(frames_np, pred, cv2)
            torch.cuda.synchronize()
            ref_s.append(time.perf_counter() - t0)
    pb_bytes = T * N * 32 + cands * 340 + T * Dt.MAX_DET * 20
    _, _, counts = Dt.person_boxes(pred, sizes, D)
    res = {'gpu': smi, 'frames': T, 'inp_dim': D, 'predictions_per_frame': N, 'person_candidates': cands,
           'survivors': int(counts.sum()),
           'letterbox_ms': [min(lb_ms), max(lb_ms)], 'letterbox_bytes': lb_bytes,
           'letterbox_GBps': [lb_bytes / max(lb_ms) / 1e6, lb_bytes / min(lb_ms) / 1e6],
           'person_boxes_ms': [min(pb_ms), max(pb_ms)], 'person_boxes_bytes': pb_bytes,
           'person_boxes_GBps': [pb_bytes / max(pb_ms) / 1e6, pb_bytes / min(pb_ms) / 1e6],
           'person_boxes_every_row_passes_ms': [min(wc_ms), max(wc_ms)],
           'video_boxes_s': [min(vb_s), max(vb_s)]}
    res['reference_flow_s'] = [min(ref_s), max(ref_s)] if ref_s else 'not measured: no cv2'
    print(json.dumps(res))


if __name__ == '__main__':
    main()
