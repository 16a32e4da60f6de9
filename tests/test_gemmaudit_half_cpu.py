"""CPU: the half form's per-launch audit (tests/gemmaudit_half.py) on synthetic plain launches: an output computed
as the device computes it (fp16 operands and weight copy, fp32 arithmetic, one fp16 rounding) passes; one moved by a
hundredth does not; the weight copy is fp16(W 2^s_W) 2^-s_W with max |W| 2^s_W in [2^14, 2^15)."""
import numpy as np
import pytest

import gemmaudit as GA
import gemmaudit_half as GAH


def _launch(relu, seed):
    rng = np.random.default_rng(seed)
    F, J, N, K = 40, 17, 64, 96
    A = rng.standard_normal((F * J, K)).astype(np.float16).astype(np.float32)
    W = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    P = dict(epi=0, N=N, relu=relu, tc_form=3, core=0, index=0, F=F, J=J, ldw=K, ld_out=N, tma_mask=1, nseg=1, fpt=7,
             bias=1, res=0, C=0, tiles_per_mask=1, segs=[dict(tap_stride=0, map=(1, 1, 1, 0))],
             res_map=(1, 1, 1, 0), heads=0, Cg=0)
    S = dict(A=A, W=W, bias=b, out0=np.zeros((F * J, N), np.float32))
    y = A @ GAH.weight_copy(W).astype(np.float32).T + b
    if relu:
        y = np.maximum(y, 0)
    return P, S, y.astype(np.float16).astype(np.float32)


@pytest.mark.parametrize('relu', [0, 1])
def test_device_arithmetic_passes_and_a_moved_output_fails(relu):
    P, S, y = _launch(relu, 3 + relu)
    assert GAH.check(P, S, y)['worst'] <= 1.0
    y[5, 7] += 0.01
    with pytest.raises(GA.AuditError):
        GAH.check(P, S, y)


def test_weight_copy():
    W = np.array([[0.3, -1e-3, 2.5e-9], [0.0, 0.1, -0.2999]], np.float32)
    c = GAH.weight_copy(W)
    s = 14 - (np.frexp(0.3)[1] - 1)
    assert 2 ** 14 <= 0.3 * 2 ** s < 2 ** 15
    assert np.array_equal(c, np.ldexp(np.ldexp(W.astype(np.float64), s).astype(np.float16).astype(np.float64), -s))
    assert np.array_equal(GAH.weight_copy(np.zeros((2, 2), np.float32)), np.zeros((2, 2)))
