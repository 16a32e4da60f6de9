"""numpy restatement of gast_pose_metrics' segment rows (csrc/pipeline.cuh), for the CPU and GPU tests of the scoring.

Test infrastructure, CPU only.  Per segment of frames the row is
    [frames, sum_f mpjpe_f, sum_f p_mpjpe_f, sum_f dist_fj for each joint j, count(dist_fj < thr_k) for each k]
with dist the float32 distance in the pinned order sqrt((dx*dx + dy*dy) + dz*dz), every step rounded (the order of
torch's CPU diff.pow(2).sum(-1).sqrt() in the reference's euclidean_losses), mpjpe_f the mean of a frame's distances
and p_mpjpe_f the float32 per-frame value of tests/pmpjperef.py's port of the Procrustes alignment.  Sums are fp64 in
numpy's order, so the last bits differ from the kernel's fixed order.
"""
import numpy as np

import pmpjperef as PR


def distances(pred, tgt):
    """(..., 3) float32 x2 -> (...) float32, sqrt((dx*dx + dy*dy) + dz*dz) rounded at every step"""
    d = np.asarray(pred, np.float32) - np.asarray(tgt, np.float32)
    sq = d * d
    return np.sqrt((sq[..., 0] + sq[..., 1]) + sq[..., 2])


def zeroed(tgt):
    """a copy of the target with joint 0 at the origin (main.py:327 inputs_3d[:, :, 0] = 0)"""
    t = np.array(tgt, np.float32)
    t[:, 0] = 0
    return t


def segment_rows(pred, tgt, seg_start, thresholds=(), zero_root=False, procrustes=True):
    pred = np.asarray(pred, np.float32)
    tgt = zeroed(tgt) if zero_root else np.asarray(tgt, np.float32)
    thr = np.asarray(thresholds, np.float32).reshape(-1)
    J = pred.shape[1]
    dist = distances(pred, tgt)
    pm = PR.p_mpjpe_per_frame(pred, tgt).astype(np.float32).astype(np.float64) if procrustes and len(pred) \
        else np.zeros(len(pred))
    rows = np.zeros((len(seg_start) - 1, 3 + J + thr.size))
    for s in range(len(seg_start) - 1):
        a, b = int(seg_start[s]), int(seg_start[s + 1])
        d = dist[a:b].astype(np.float64)
        rows[s, 0] = b - a
        rows[s, 1] = d.mean(1).sum()
        rows[s, 2] = pm[a:b].sum()
        rows[s, 3:3 + J] = d.sum(0)
        rows[s, 3 + J:] = [(dist[a:b] < t).sum() for t in thr]
    return rows
