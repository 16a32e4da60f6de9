"""Device-side counterpart of the reference's common/loss.py (same names and signatures; lives under
`device.` so that it does not shadow the reference module): `mpjpe` (loss.py:5-11), `p_mpjpe` (loss.py:14-53),
`euclidean_losses`, `pck` and `auc` (loss.py:56-90) on the device (gast_b200/pipeline.py, csrc/pipeline.cuh).
`mpjpe` is differentiable (forward and backward come from one kernel pass); the others take numpy arrays like the
reference (main.py:281-283) or CUDA tensors.  `euclidean_losses`, `pck` and `auc` take 3D points (..., J, 3) with
J <= 32; their distances are the reference's float32 ones bit for bit, so `pck` counts the same points."""
import numpy as np
import torch

from gast_b200 import pipeline as _P


def _cuda(x):
    if isinstance(x, torch.Tensor):
        return x
    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).cuda()


def mpjpe(predicted, target):
    assert predicted.shape == target.shape
    return _P.mpjpe(predicted, target)


def p_mpjpe(predicted, target):
    assert predicted.shape == target.shape
    as_numpy = not isinstance(predicted, torch.Tensor)
    if as_numpy:
        predicted = torch.as_tensor(np.ascontiguousarray(predicted, dtype=np.float32)).cuda()
        target = torch.as_tensor(np.ascontiguousarray(target, dtype=np.float32)).cuda()
    m = _P.p_mpjpe_per_frame(predicted, target).mean()
    return np.float32(m.item()) if as_numpy else m


def _counts(actual, target, thresholds, distances=False):
    """one gast_pose_metrics launch over all points as one segment: (counts below each threshold, points[, dist])"""
    assert tuple(actual.shape) == tuple(target.shape), 'input tensors must have the same size'
    a, t = _cuda(actual), _cuda(target)
    J = int(a.shape[-2]) if a.dim() >= 2 else 0
    a3, t3 = a.reshape(-1, J, 3), t.reshape(-1, J, 3)
    N = int(a3.shape[0])
    out = _P.pose_metrics(a3, t3, [0, N], thresholds, procrustes=False, distances=distances)
    rows, dist = out if distances else (out, None)
    counts = rows[0, 3 + J:].cpu().tolist()
    return counts, N * J, (dist.reshape(a.shape[:-1]) if distances else None)


def euclidean_losses(actual, target):
    """(..., J, 3) x2 -> (..., J) CUDA float32: the distance of every point, sqrt((dx*dx + dy*dy) + dz*dz)"""
    return _counts(actual, target, (), distances=True)[2]


def pck(actual, expected, threshold=150):
    """the fraction of points closer than `threshold` (Python float, count / points in double)"""
    counts, n, _ = _counts(actual, expected, [threshold])
    return counts[0] / n


def auc(actual, expected):
    """the mean of pck over torch.linspace(0, 150, 31), the thresholds of mpii_compute_3d_pck.m, from one launch"""
    thresholds = torch.linspace(0, 150, 31).tolist()
    counts, n, _ = _counts(actual, expected, thresholds)
    return torch.tensor([c / n for c in counts], dtype=torch.float64).mean().item()
