"""The tensor-core GEMM core's tile order (csrc/gemm_tc.cuh): one CTA per tile on a 1D grid, the column tile the
fast index.  One GEMM through gast_debug_gemm (core 0) at tile counts below, at, just above and many times the SM
count (so tiles run in several waves), at 1 to 7 ring stages per tile, with partial / several column tiles and a
partial last row tile, against fp64 at the 3xTF32 bar and bitwise equal between two runs; a GEMM's rows do not depend
on how many tiles the launch has; and the global-attention epilogue, whose scratch is the ring, at many tiles: the
single-head kind, and MultiGlobalGraph at J > MIX_JMAX, against the torch-CPU port of the reference."""
import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth

pytestmark = pytest.mark.gpu

BM, BN = 128, 128      # tile of gemm_tc.cuh


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _gemm(lib, a, w, M, N, K):
    o = torch.full((M, N), float('nan'), dtype=torch.float32, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, 0, 0, None,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return o


def _inputs(M, N, K, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    a = torch.randn(M, K, device='cuda', generator=g)
    w = torch.randn(N, K, device='cuda', generator=g) / np.sqrt(K)
    return a, w


def _check(lib, M, N, K, seed, what):
    a, w = _inputs(M, N, K, seed)
    o1 = _gemm(lib, a, w, M, N, K)
    o2 = _gemm(lib, a, w, M, N, K)
    ref = a.double() @ w.double().T
    d = o1.double() - ref
    rel = float(torch.sqrt((d ** 2).mean()) / torch.sqrt((ref ** 2).mean()))
    assert bool(torch.isfinite(o1).all()) and rel < 2e-6, (what, M, N, K, rel)
    assert torch.equal(o1, o2), (what, M, N, K)
    return o1


@pytest.mark.parametrize('tiles', ['below', 'equal', 'above', 'many'])
def test_tc_tile_count(tiles):
    """One column tile (N = 4), so the tile count is the row-tile count; the last row tile is partial."""
    lib = _lib.load()
    s = _sms()
    nt = {'below': s - 1, 'equal': s, 'above': s + 1, 'many': 4 * s + 3}[tiles]
    M = BM * (nt - 1) + 77
    _check(lib, M, 4, 32 * 5, 11 + nt, tiles)


@pytest.mark.parametrize('stages', [1, 2, 4, 5, 7])
@pytest.mark.parametrize('N', [132, 1024])
def test_tc_stages_per_tile(stages, N):
    """About three waves of tiles at every stage count, including counts that are not multiples of the ring's slots."""
    lib = _lib.load()
    col_tiles = (N + BN - 1) // BN
    row_tiles = (3 * _sms()) // col_tiles + 2
    M = BM * (row_tiles - 1) + 45
    _check(lib, M, N, 32 * stages, 100 * stages + N, 'stages')


def test_tc_schedule_independence():
    """The first rows of a GEMM of several waves of tiles, recomputed by a GEMM of less than one wave, are bitwise
    the same."""
    lib = _lib.load()
    s = _sms()
    N, K = 1024, 32 * 7
    col_tiles = N // BN
    big_rows = BM * (5 * s // col_tiles) + 19           # ~5 waves, partial last row tile
    small_rows = BM * (s // col_tiles)                  # at most one wave
    assert (big_rows + BM - 1) // BM * col_tiles > 4 * s and small_rows // BM * col_tiles <= s
    a, w = _inputs(big_rows, N, K, 5)
    big = _check(lib, big_rows, N, K, 5, 'big')
    small = _gemm(lib, a[:small_rows].contiguous(), w, small_rows, N, K)
    assert torch.equal(big[:small_rows], small)


def _tc_launches(m):
    h = list(m.__dict__['_gast_handles'].values())[0]
    return int(h.lib.gast_last_tc_launch_count(h.h))


def _chain_adj(J):
    a = torch.eye(J)
    for j in range(1, J):
        a[j, j - 1] = a[j - 1, j] = 1.0
    return a


@pytest.mark.parametrize('kind', ['single_head_j17', 'multi_head_j24'])
def test_tc_global_epilogue_many_tiles(kind):
    """The global-mix epilogue on the tensor-core core (the single-head kind; MultiGlobalGraph for J > MIX_JMAX = 20)
    at several waves of tiles."""
    from model.global_attention import GlobalGraph, MultiGlobalGraph
    from oracle import gast_torch_ref as TR
    engine.set_gemm_core(0)
    s = _sms()
    if kind == 'single_head_j17':
        J, C, fpt = 17, 32, 128 // 17
        BT = 4 * s * fpt + 5                               # > 4 waves (one column tile), a partial last tile
        m = GlobalGraph(_chain_adj(J), C, 8)
        synth.randomize_module(m, 31)
        x = torch.from_numpy(synth.synth_input(1, BT * C, J, 1, seed=32)).reshape(BT, C, J).contiguous()
        ref = TR.global_graph(x, {k: v.clone() for k, v in m.state_dict().items()}, '')
    else:
        J, C, fpt = 24, 32, 128 // 24
        B, T = 4, (3 * s * fpt) // 4 + 3                  # > 3 waves
        m = MultiGlobalGraph(_chain_adj(J), C, 8, dropout=0.05)
        synth.randomize_module(m, 41)
        x = torch.from_numpy(synth.synth_input(B, T * C, J, 1, seed=42)).reshape(B, T, C, J).permute(0, 1, 3, 2)
        x = x.contiguous()
        ref = TR.multi_global_graph(x, {k: v.clone() for k, v in m.state_dict().items()}, '')
    m = m.cuda().eval()
    with torch.no_grad():
        y1 = m(x.cuda())
        assert _tc_launches(m) > 0
        y2 = m(x.cuda())
    assert torch.equal(y1, y2), kind
    err = float((y1.cpu() - ref).abs().max())
    assert err < 1e-4, (kind, err)
