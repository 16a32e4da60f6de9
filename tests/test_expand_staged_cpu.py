"""CPU emulation of the index arithmetic of the staged expand kernel in csrc/kernels_hbm.cuh (the kernel itself is
checked on the GPU by the parity suite): the gather index ((b*T + t*stride + kk)*J + j)*Fin + i that fills the staged
rows is the input window of the strided (k,1) convolution it implements (gast_net.py:163-164), and the blocks of the
1024-channel chunks (blockIdx.y) write every output channel of their rows exactly once.  These tests check the scheme,
not the kernel source: a slip in the kernel's offsets is caught on the GPU by the 1056-channel case of
tests/test_gpu_parity.py::test_against_oracle_random_shapes."""
import numpy as np
import pytest

EXS_ROWS, EXS_THREADS = 128, 256
EXS_CHUNK = 4 * EXS_THREADS


@pytest.mark.parametrize('taps,Fin,stride,T,J', [(3, 2, 3, 27, 17), (3, 2, 1, 9, 5), (5, 2, 5, 25, 4)])
def test_expand_rows_gather_index(taps, Fin, stride, T, J):
    rng = np.random.default_rng(0)
    B = 3
    T0 = (T - taps) // stride + 1
    x = rng.standard_normal((B, T, J, Fin)).astype(np.float32)
    flat = x.reshape(-1)
    rows = B * T0 * J
    KF = taps * Fin
    for row in rng.integers(0, rows, 64):
        f, j = divmod(int(row), J)
        b, t = divmod(f, T0)
        got = [flat[((b * T + t * stride + k // Fin) * J + j) * Fin + k % Fin] for k in range(KF)]
        want = x[b, t * stride:t * stride + taps, j, :].reshape(-1)
        assert np.array_equal(np.array(got, np.float32), want)


@pytest.mark.parametrize('C', [4, 128, 1020, 1024, 1056, 2112, 4096])
@pytest.mark.parametrize('nrows', [EXS_ROWS, 37])
def test_expand_rows_channel_chunks_cover_each_output_once(C, nrows):
    hits = np.zeros((nrows, C), np.int32)
    for by in range((C + EXS_CHUNK - 1) // EXS_CHUNK):      # grid.y = cdiv(C, EXS_CHUNK)
        c0 = by * EXS_CHUNK
        cq = min(C - c0, EXS_CHUNK) >> 2
        rpp = EXS_THREADS // cq
        for tid in range(EXS_THREADS):
            cg, rsub = tid % cq, tid // cq
            if rsub >= rpp:
                continue
            c = c0 + cg * 4
            hits[rsub:nrows:rpp, c:c + 4] += 1
    assert (hits == 1).all()
