"""The activation feed and the plain store of the tensor-core GEMM core (csrc/gemm_tc.cuh): segments whose tile rows
are contiguous in their source arrive as one 128-byte-swizzled TMA box per stage, and the plain epilogue stores the
tile by TMA with a map whose dims drop rows past the GEMM's and whose box height keeps a frame-aligned tile inside its
own frames.

- gast_debug_gemm in each precision with an output buffer longer than M: the rows after M keep their NaN sentinels,
  and the result is within the form's emulation and fp64 bars, bitwise equal between two runs;
- an output 4, 8 or 12 bytes into a buffer, which the tensor store's map cannot take: refused before any launch;
- a SpatioTemporalModel at J = 17 (119-row frame tiles, several per GEMM; identity-map layers fed by TMA, the stage
  convolutions gathered per row): the tensor-core forward matches the FFMA core's to the parity bar and is bitwise
  equal between two runs."""
import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth
import f16x3ref as F
import tf32ref as R

pytestmark = pytest.mark.gpu

MODES = {'f16x3': 0, 'tf32': 1, '3xtf32': 3}
PAD_ROWS = 200


def _gemm(a, w, M, N, K, tc_mode):
    lib = _lib.load()
    o = torch.full((M + PAD_ROWS, N), float('nan'), dtype=torch.float32, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, tc_mode, 0, None,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return o.cpu().numpy()


@pytest.mark.parametrize('K', [32, 96, 1536])
@pytest.mark.parametrize('N', [4, 132, 516])
@pytest.mark.parametrize('M', [300, 128 * 3])
@pytest.mark.parametrize('prec', list(MODES))
def test_rows_past_m_untouched(prec, M, N, K):
    rs = np.random.RandomState(M + 7 * N + K)
    A = rs.standard_normal((M, K)).astype(np.float32)
    W = (rs.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    a, w = torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda()
    o1 = _gemm(a, w, M, N, K, MODES[prec])
    o2 = _gemm(a, w, M, N, K, MODES[prec])
    assert np.isnan(o1[M:]).all() and np.isnan(o2[M:]).all()
    y = o1[:M]
    assert np.isfinite(y).all()
    assert np.array_equal(y.view(np.uint32), o2[:M].view(np.uint32))
    exact = A.astype(np.float64) @ W.astype(np.float64).T
    if prec == 'f16x3':
        emu = F.gemm(A, W).astype(np.float64)
    elif prec == '3xtf32':
        emu = F.gemm_3xtf32(A, W).astype(np.float64)
    else:
        emu = R.tf32(A).astype(np.float64) @ R.tf32(W).astype(np.float64).T
    rel = lambda ref: float(np.linalg.norm(y - ref) / np.linalg.norm(ref))
    assert rel(emu) < 2e-6, (prec, M, N, K, rel(emu))
    assert rel(exact) < (2e-3 if prec == 'tf32' else 2e-6), (prec, M, N, K, rel(exact))


@pytest.mark.parametrize('offset', [4, 8, 12])
@pytest.mark.parametrize('prec', list(MODES))
def test_unaligned_output_refused_up_front(prec, offset):
    """the plain store's tensor map needs a 16-byte-aligned output: the tensor-core core does not take an output 4, 8
    or 12 bytes into a buffer (tc_supported), so the call is refused before any launch and the buffer is untouched"""
    lib = _lib.load()
    M, N, K = 300, 36, 64
    a = torch.ones((M, K), dtype=torch.float32, device='cuda')
    w = torch.ones((N, K), dtype=torch.float32, device='cuda')
    o = torch.full((M * N + 8,), float('nan'), dtype=torch.float32, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr() + offset, M, N, K, 0, MODES[prec], 0, None,
                             torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc != 0 and 'not supported by the tensor-core core' in _lib.last_error(), _lib.last_error()
    assert torch.isnan(o).all()


def _adj(J):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))


def test_frame_tiles_match_ffma():
    from model.gast_net import SpatioTemporalModel
    J = 17
    m = SpatioTemporalModel(_adj(J), J, 2, J, [3, 3, 3], channels=64)
    synth.randomize_module(m, 11)
    m = m.cuda().eval()
    x = torch.from_numpy(synth.synth_input(12, 27, J, 2, seed=3)).cuda()
    h = None
    try:
        with torch.no_grad():
            y1 = m(x).cpu().numpy()
            h = list(m.__dict__['_gast_handles'].values())[0]
            assert int(h.lib.gast_last_tc_launch_count(h.h)) > 0
            y2 = m(x).cpu().numpy()
            engine.set_gemm_core(1)
            yf = m(x).cpu().numpy()
            assert int(h.lib.gast_last_tc_launch_count(h.h)) == 0
    finally:
        engine.set_gemm_core(0)
    assert np.array_equal(y1.view(np.uint32), y2.view(np.uint32))
    assert np.abs(y1 - yf).max() < 1e-4
