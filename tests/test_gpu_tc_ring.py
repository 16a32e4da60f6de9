"""The tensor-core GEMM core's shared-memory ring (csrc/gemm_tc.cuh): one GEMM through gast_debug_gemm (core 0) at
K lengths that reach every phase of the producer / consumer ring (fewer stages than slots, one short of a full ring,
exactly full, one wrap, two wraps, many), with a partial last row tile and partial / several column tiles, against
fp64 at the 3xTF32 bar and bitwise equal between two runs."""
import numpy as np
import pytest
import torch

from gast_b200 import _lib

pytestmark = pytest.mark.gpu

TC_STAGES = 3          # ring slots of gemm_tc.cuh


def _gemm(lib, a, w, M, N, K):
    o = torch.full((M, N), float('nan'), dtype=torch.float32, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, 0, 0, None,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return o.cpu().numpy()


@pytest.mark.parametrize('stages', sorted({1, TC_STAGES - 1, TC_STAGES, TC_STAGES + 1, 2 * TC_STAGES + 1, 48}))
@pytest.mark.parametrize('N', [4, 132, 256])
def test_tc_ring_phases(stages, N):
    lib = _lib.load()
    M, K = 300, 32 * stages
    rs = np.random.RandomState(1000 * stages + N)
    A = rs.standard_normal((M, K)).astype(np.float32)
    W = (rs.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    a, w = torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda()
    o1 = _gemm(lib, a, w, M, N, K)
    o2 = _gemm(lib, a, w, M, N, K)
    ref = A.astype(np.float64) @ W.astype(np.float64).T
    d = o1.astype(np.float64) - ref
    rel = np.sqrt((d ** 2).mean()) / np.sqrt((ref ** 2).mean())
    assert np.isfinite(o1).all() and rel < 2e-6, (stages, N, rel)
    assert np.array_equal(o1, o2), (stages, N)
