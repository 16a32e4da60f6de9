"""The weight feed of the tensor-core GEMM core (csrc/gemm_tc.cuh): every copy's TMA map describes a stage as rows of
2 KB (a k-quad or k-octet of a 128-column tile), and elements past the copy's N columns read as zero.  One GEMM
through gast_debug_gemm (core 0) in each precision (tc_mode 0 F16X3, 1 1xTF32, 3 3xTF32) at column counts with
partial first and last column tiles and one to many column tiles, and at K of one, three and 48 stages: against the
form's emulation (tests/f16x3ref.py, tests/tf32ref.py) and against fp64, bitwise equal between two runs."""
import numpy as np
import pytest
import torch

from gast_b200 import _lib
import f16x3ref as F
import tf32ref as R

pytestmark = pytest.mark.gpu

MODES = {'f16x3': 0, 'tf32': 1, '3xtf32': 3}


def _gemm(a, w, M, N, K, tc_mode):
    lib = _lib.load()
    o = torch.full((M, N), float('nan'), dtype=torch.float32, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, tc_mode, 0, None,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return o.cpu().numpy()


def _col_l2(y, ref):
    """the largest relative L2 error of an output column (a wrong or unfilled column of W shows in its own column)"""
    d = np.asarray(y, np.float64) - ref
    return float((np.linalg.norm(d, axis=0) / np.linalg.norm(ref, axis=0)).max())


@pytest.mark.parametrize('K', [32, 96, 1536])
@pytest.mark.parametrize('N', [4, 36, 124, 128, 132, 260, 516, 2048])
@pytest.mark.parametrize('prec', list(MODES))
def test_weight_rows(prec, N, K):
    M = 300                                       # a partial last row tile
    rs = np.random.RandomState(7 * N + K)
    A = rs.standard_normal((M, K)).astype(np.float32)
    W = (rs.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    a, w = torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda()
    o1 = _gemm(a, w, M, N, K, MODES[prec])
    o2 = _gemm(a, w, M, N, K, MODES[prec])
    assert np.isfinite(o1).all()
    assert np.array_equal(o1.view(np.uint32), o2.view(np.uint32))
    exact = A.astype(np.float64) @ W.astype(np.float64).T
    if prec == 'f16x3':
        emu = F.gemm(A, W).astype(np.float64)
    elif prec == '3xtf32':
        emu = F.gemm_3xtf32(A, W).astype(np.float64)
    else:
        emu = R.tf32(A).astype(np.float64) @ R.tf32(W).astype(np.float64).T
    e_emu, e_exact = _col_l2(o1, emu), _col_l2(o1, exact)
    assert e_emu < 2e-6, (prec, N, K, e_emu)      # the form's own products, fp32 accumulation
    if prec == 'tf32':
        assert e_exact < 2e-3, (N, K, e_exact)    # TF32 operand rounding
    else:
        assert e_exact < 2e-6, (prec, N, K, e_exact)   # the fp32-grade bar


def test_debug_gemm_modes():
    """tc_mode 3 runs 3xTF32; the modes between and past the offered ones, and the FFMA core with a tensor-core
    mode, are refused"""
    lib = _lib.load()
    a = torch.zeros((128, 32), device='cuda')
    w = torch.zeros((32, 32), device='cuda')
    o = torch.full((128, 32), float('nan'), device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    assert lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), 128, 32, 32, 0, 3, 0, None, st) == 0
    torch.cuda.synchronize()
    assert (o.cpu().numpy() == 0).all()
    for core, mode in ((0, 2), (0, 4), (1, 3)):
        assert lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), 128, 32, 32, core, mode, 0, None, st) != 0
        assert 'tc_mode' in _lib.last_error()
