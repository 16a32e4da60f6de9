"""CPU checks of tests/tf32wgradref.py, the emulation the GPU tests hold the TF32 weight-gradient kernel to: its
rounding is the tf32 rounding of tests/tf32ref.py bit for bit, its result lies within the TF32 bound of the exact
contraction, and its row splits are dense_tn's."""
import numpy as np
import pytest

import tf32ref
import tf32wgradref as W
from test_gpu_grad_exact import dense_tn_split


def test_rounding_bit_equal_to_tf32ref():
    rs = np.random.RandomState(0)
    bits = rs.randint(0, 2 ** 32, size=1 << 20, dtype=np.uint64).astype(np.uint32)
    # ties (low 13 bits exactly 0x1000), values next to them, subnormals, the largest finite values, zeros, inf
    special = np.array([0x1000, 0x0FFF, 0x1001, 0x3F801000, 0xBF801000, 0x3F800FFF, 0x00000001, 0x00001000,
                        0x007FF000, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0x7F7FF000, 0xFF7FF000, 0x00000000,
                        0x80000000, 0x7F800000, 0xFF800000], dtype=np.uint32)
    x = np.concatenate([bits, special]).view(np.float32)
    x = x[~np.isnan(x)]
    a, b = W.tf32(x), tf32ref.tf32(x)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize('M,N,K', [(1, 32, 32), (33, 64, 96), (2176, 128, 384), (5000, 96, 64)])
def test_within_tf32_bound_of_fp64(M, N, K):
    rs = np.random.RandomState(M + N + K)
    dZ = rs.standard_normal((M, N)).astype(np.float32)
    A = (rs.standard_normal((M, K)) * 3.0).astype(np.float32)
    got = W.wgrad(dZ, A, 132).astype(np.float64)
    exact = dZ.astype(np.float64).T @ A.astype(np.float64)
    err = np.abs(got - exact)
    assert (err <= W.bound(dZ, A, 132)).all()
    # and the rounding is there: unrounded operands would be ~1e3x closer
    rel = np.linalg.norm(got - exact) / np.linalg.norm(exact)
    assert 1e-5 < rel < 1e-3, rel


@pytest.mark.parametrize('M', [1, 15, 16, 17, 255, 256, 2176, 6528, 19584, 58752, 626688, 626689])
@pytest.mark.parametrize('N,K', [(8, 128), (128, 128), (256, 384), (1024, 1536), (64, 8)])
@pytest.mark.parametrize('sms', [132, 114])
def test_split_matches_dense_tn(M, N, K, sms):
    S, rps = W.split(M, N, K, sms)
    assert (S, rps) == dense_tn_split(M, N, K, sms)
    assert rps % W.WG_M == 0 and (S - 1) * rps < M <= S * rps
