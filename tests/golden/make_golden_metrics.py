"""Golden joint distances, PCK and AUC from the UNMODIFIED reference (/root/reference common/loss.py:56-90
euclidean_losses, pck, auc; float32 torch tensors on the CPU).

Run where an original checkout is at hand (found as oracle/make_ref.py finds it, or given as the argument):
    python tests/golden/make_golden_metrics.py [<original GAST-Net checkout>]
Writes tests/golden/metrics_17.npz (and nothing else): per case the float32 inputs (N,17,3), the reference's
distances (N,17), its squared distances before the square root (euclidean_losses' own first two steps,
diff.pow(2).sum(-1), which the function does not return), its pck at every threshold of THRESHOLDS and its auc.  The cases put distances exactly on
thresholds (integer targets moved by multiples of 5 along one axis, or of (3,4,0)) and hold degenerate frames.
"""
import os
import sys
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import make_ref                                                         # noqa: E402
REF = make_ref.find_reference(sys.argv[1] if len(sys.argv) > 1 else None)
assert REF, 'no original GAST-Net checkout found'

sys.path.insert(0, REF)
from common.loss import euclidean_losses, pck, auc                                 # noqa: E402
import common.loss as _ref_loss                                                     # noqa: E402
assert _ref_loss.__file__.startswith(REF), _ref_loss.__file__

J = 17
THRESHOLDS = np.array([0.0, 2.5, 5.0, 10.0, 37.5, 50.0, 100.0, 145.0, 150.0, 1e-3], np.float32)


def cases():
    rs = np.random.RandomState(17)
    out = {}
    t = rs.uniform(-800, 800, (64, J, 3))
    out['random'] = (t + rs.standard_normal((64, J, 3)) * rs.uniform(1, 120, (64, J, 1)), t)
    # integer targets, the prediction k*5 mm away along one axis (or k*(3,4,0)): dist = 5k exactly, on the thresholds
    t = rs.randint(-1000, 1000, (62, J, 3)).astype(np.float64)
    k = rs.randint(0, 31, (62, J))
    off = np.zeros((62, J, 3))
    axis = rs.randint(0, 4, (62, J))
    for a in range(3):
        off[..., a] = np.where(axis == a, 5.0 * k, 0.0)
    off[..., 0] += np.where(axis == 3, 3.0 * k, 0.0)
    off[..., 1] += np.where(axis == 3, 4.0 * k, 0.0)
    out['on_threshold'] = (t + off * np.where(rs.rand(62, J, 1) < 0.5, 1.0, -1.0), t)
    # degenerate frames: an exact copy, every joint at one point, all zeros, one joint far away
    t = rs.uniform(-500, 500, (4, J, 3))
    p = t.copy()
    p[1] = p[1, :1]
    t[1] = t[1, :1]
    p[2] = 0
    t[2] = 0
    p[3, 5] += 1e4
    out['degenerate'] = (p, t)
    return {k: (np.asarray(p, np.float32), np.asarray(t, np.float32)) for k, (p, t) in out.items()}


def main():
    out = {'thresholds': THRESHOLDS}
    for name, (p, t) in cases().items():
        a, e = torch.from_numpy(p), torch.from_numpy(t)
        out[name + '_pred'], out[name + '_tgt'] = p, t
        out[name + '_dist'] = euclidean_losses(a, e).numpy()
        out[name + '_dist_sq'] = (a - e).pow(2).sum(-1, keepdim=False).numpy()
        out[name + '_pck'] = np.array([pck(a, e, threshold=float(th)) for th in THRESHOLDS], np.float64)
        out[name + '_auc'] = np.float64(auc(a, e))
    np.savez_compressed(os.path.join(HERE, 'metrics_17.npz'), **out)
    print('metrics_17', {k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
