"""The fp32-grade inference form of the tensor-core core (three fp16 products on power-of-two-scaled operands,
csrc/gemm_tc.cuh), emulated in numpy (tests/f16x3ref.py): as close to fp64 as the 3xTF32 form over fp32's range,
with every scaled operand inside fp16's range and every unscale factor a normal fp32."""
import numpy as np
import pytest

import f16x3ref as F

FACTOR = 4.0        # F16X3 error / 3xTF32 error allowed (both are 22-bit splits; measured 0.6 - 1.6)
FLOOR = 1e-7        # ... or an error below a few fp32 ulps


def _row_err(y, ref):
    """max over rows of the row's relative L2 error (rows span many decades, so each is measured on its own)"""
    y = np.asarray(y, np.float64)
    n = np.linalg.norm(ref, axis=1)
    keep = n > 0
    return float((np.linalg.norm(y - ref, axis=1)[keep] / n[keep]).max())


def _check(A, W):
    A, W = np.asarray(A, np.float32), np.asarray(W, np.float32)
    ref = A.astype(np.float64) @ W.astype(np.float64).T
    e16, e32 = _row_err(F.gemm(A, W), ref), _row_err(F.gemm_3xtf32(A, W), ref)
    assert e16 <= max(FACTOR * e32, FLOOR), (e16, e32)
    _check_ranges(A, W)
    return e16, e32


def _check_ranges(A, W):
    wh, wl, sw = F.split_w(W)
    ah, al, s = F.split_a(A, sw)
    for x in (wh, wl, ah, al):
        assert np.isfinite(x).all() and np.abs(x.astype(np.float32)).max() <= F.F16_MAX
    e = -(s + sw)
    assert (e >= -126).all() and (e <= 127).all()       # 2^-(s_r + s_W) is a normal fp32
    assert (s >= -126).all() and (s <= 127).all()       # and so is 2^s_r


def _w(rs, N, K, scale=1.0):
    return (rs.standard_normal((N, K)) / np.sqrt(K) * scale).astype(np.float32)


@pytest.mark.parametrize('K', [32, 64, 96, 160, 512, 1536])
def test_k_lengths(K):
    rs = np.random.RandomState(K)
    _check(rs.standard_normal((24, K)), _w(rs, 20, K))


def test_rows_from_1e_minus30_to_1e30():
    rs = np.random.RandomState(1)
    M, K = 61, 256
    A = rs.standard_normal((M, K)) * 10.0 ** np.linspace(-30, 30, M)[:, None]
    _check(A, _w(rs, 16, K))


def test_rows_mixing_1e_minus6_and_1e6_in_one_stage():
    rs = np.random.RandomState(2)
    M, K = 32, 128
    A = rs.standard_normal((M, K)) * np.where(rs.uniform(size=(M, K)) < 0.5, 1e-6, 1e6)
    _check(A, _w(rs, 16, K))


@pytest.mark.parametrize('scale', [1e-20, 1e20])
def test_weights_scaled(scale):
    rs = np.random.RandomState(3)
    K = 192
    _check(rs.standard_normal((16, K)), _w(rs, 24, K, scale))


def test_zero_rows_and_subnormal_inputs():
    rs = np.random.RandomState(4)
    M, K = 16, 128
    A = rs.standard_normal((M, K)).astype(np.float32)
    A[3] = 0
    A[5, :64] = 0                                           # a zero stage in a row
    sub = (rs.standard_normal((M, K)) * 1e-40).astype(np.float32)
    assert (np.abs(sub[sub != 0]) < np.finfo(np.float32).tiny).all()
    A[7:9] = np.where(rs.uniform(size=(2, K)) < 0.5, sub[7:9], A[7:9])   # subnormals among normal values
    A[10] = sub[10]                                                       # a row of subnormals only
    W = _w(rs, 16, K)
    y = F.gemm(A, W)
    assert (y[3] == 0).all()
    ref = A.astype(np.float64) @ W.astype(np.float64).T
    normal = [i for i in range(M) if i != 10]
    e16, e32 = _row_err(y[normal], ref[normal]), _row_err(F.gemm_3xtf32(A, W)[normal], ref[normal])
    assert e16 <= max(FACTOR * e32, FLOOR), (e16, e32)
    # the subnormal-only row: the clamp keeps 2^-(s_r + s_W) a normal fp32, so the row is scaled short of
    # [2^14, 2^15) and its fp16 split loses bits (3.5e-41 on outputs of ~1e-40); the error stays below 1/64 of the
    # smallest normal fp32
    assert np.abs(y[10] - ref[10]).max() < np.finfo(np.float32).tiny / 64
    _check_ranges(A, W)


def test_zero_and_tiny_weights():
    rs = np.random.RandomState(5)
    A = rs.standard_normal((8, 64)).astype(np.float32)
    assert (F.gemm(A, np.zeros((8, 64), np.float32)) == 0).all()
    W = np.full((8, 64), 1e-42, np.float32)                  # a subnormal weight matrix: s_W beyond 127
    assert F.w_scale(W) > 127
    _check_ranges(A, W)


def test_non_finite_inputs_become_nan():
    rs = np.random.RandomState(6)
    A = rs.standard_normal((4, 32)).astype(np.float32)
    A[1, 3] = np.inf
    A[2, 5] = np.nan
    y = F.gemm(A, _w(rs, 8, 32))
    assert np.isnan(y[1]).all() and np.isnan(y[2]).all() and np.isfinite(y[[0, 3]]).all()


def test_scale_rule():
    """the row max lands in [2^14, 2^15) and the split carries 22 bits"""
    rs = np.random.RandomState(7)
    A = (rs.standard_normal((50, 64)) * np.exp(rs.uniform(-40, 40, (50, 1)))).astype(np.float32)
    h, lo, s = F.split_a(A, 14)
    m = np.abs(A * np.repeat(F.pow2(s), 32, axis=1)).reshape(50, 2, 32).max(axis=2)
    assert ((m >= 2.0 ** 14) & (m < 2.0 ** 15)).all()
    x = A.astype(np.float64) * np.repeat(2.0 ** s, 32, axis=1)
    r = np.abs(h.astype(np.float64) + lo.astype(np.float64) - x) / np.abs(x).reshape(50, 2, 32).max(axis=2).repeat(32, 1)
    assert r.max() < 2.0 ** -22
