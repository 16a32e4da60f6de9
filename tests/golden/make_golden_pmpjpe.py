"""Golden P-MPJPE values of degenerate frames from the UNMODIFIED reference (/root/reference common/loss.p_mpjpe, float32
numpy, one frame per call).

Run in the build container only (the GPU box has no /root/reference):
    python tests/golden/make_golden_pmpjpe.py
Writes tests/golden/pmpjpe_degenerate.npz (and nothing else): per kind of frame (tests/pmpjperef.py::frames) the
float32 inputs and the reference's per-frame errors.
"""
import os
import sys
import types
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'

sys.modules['torchsummary'] = types.SimpleNamespace(summary=None)
sys.path.insert(0, REF)
sys.path.insert(1, os.path.dirname(HERE))              # tests/, for pmpjperef.frames

from common.loss import p_mpjpe                                                     # noqa: E402
import common.loss as _ref_loss                                                     # noqa: E402
assert _ref_loss.__file__.startswith(REF), _ref_loss.__file__
from pmpjperef import frames                                                        # noqa: E402

KINDS = ('ordinary', 'planar_pred', 'planar_tgt', 'planar_tgt_rot', 'collinear_tgt', 'collinear_pred', 'reflected')


def main():
    out = {}
    for i, kind in enumerate(KINDS):
        p, t = frames(kind, 8, 17, seed=300 + i)
        out[kind + '_pred'], out[kind + '_tgt'] = p, t
        out[kind + '_per_frame'] = np.array([p_mpjpe(p[n:n + 1].copy(), t[n:n + 1].copy()) for n in range(len(p))],
                                            np.float64)
    np.savez_compressed(os.path.join(HERE, 'pmpjpe_degenerate.npz'), **out)
    print('pmpjpe_degenerate', {k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
