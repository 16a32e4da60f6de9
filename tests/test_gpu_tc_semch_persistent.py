"""GPU: the tensor-core core's SemCH GEMMs as a persistent tile loop (csrc/gemm_tc.cuh, tc_store_semch).

EPI_SEMCH launches run min(tiles, SMs) CTAs, each walking its tiles in the column-fast order, and mix each row's
neighbours on the wgmma fragments through a staging buffer that the next tile's K loop does not touch.
  * Schedule independence: the headline model's poses of its first 8 clips are bitwise the same whether the forward
    runs 4096 clips (each SM runs many SemCH tiles) or those 8 clips alone (less than one wave), at the default
    precision (F16X3) and in TF32.  Every kernel of the forward is row-wise, so a tile's result must not depend on how
    many tiles its CTA ran before it.
  * Edge shapes under the GEMM audit (tests/gemmaudit.py: every launch against fp64 of its own operands, unowned
    columns bitwise unchanged): LocalGraph at C = 96 (a half-empty second column tile per mask, whose stores must not
    reach the other mask's columns), 32 and 64, J = 15, 16, 19 and 20; SemCHGraphConv (one mask, no ReLU); tile counts
    below, at, just above and several times the SM count, with a partial last row tile; F16X3 and 1xTF32.
"""
import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth
import gemmaudit as GA

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _handles(m):
    return list(m.__dict__['_gast_handles'].values())


def _forward(m, x):
    with torch.no_grad():
        return m(x).clone()


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
def test_semch_schedule_independence(prec):
    from test_gpu_forward_fp64 import HEADLINE, HEADLINE_B, build_model
    engine.set_gemm_core(0)
    m = engine.set_precision(build_model(*HEADLINE, seed=1).cuda(), prec)
    x = torch.from_numpy(synth.synth_input(HEADLINE_B, 27, 17, 2, seed=1234)).cuda()
    big = _forward(m, x)
    small = _forward(m, x[:8].contiguous())
    assert bool(torch.isfinite(big).all())
    assert torch.equal(big[:8], small), float((big[:8] - small).abs().max())


def _audited(m, x, prec):
    """m(x) with the GEMM audit on every handle of m; the SemCH records of the tensor-core core"""
    engine.set_gemm_core(0)
    engine.set_precision(m, prec)
    y0 = _forward(m, x)                              # creates the handle
    aud = GA.Auditor()
    for h in _handles(m):
        aud.install(h.lib, h.h)
    try:
        y1 = _forward(m, x)
        torch.cuda.synchronize()
    finally:
        for h in _handles(m):
            h.lib.gast_debug_set_gemm_audit(h.h, _lib.GemmAuditFn(), None)
    assert aud.failure is None, aud.failure
    assert torch.equal(y0, y1)
    recs = [r for r in aud.records if r['epi'] == 'semch']
    assert recs and all(r['core'] == 'tc' and r['form'] == {'fp32': 'f16x3', 'tf32': 'tf32'}[prec] for r in recs), recs
    return recs


def _tiles(rec, fpt):
    return -(-rec['F'] // fpt) * (rec['N'] // 128)


def _x(shape, seed):
    return torch.from_numpy((0.7 * np.random.RandomState(seed).standard_normal(shape)).astype(np.float32)).cuda()


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
@pytest.mark.parametrize('tiles', ['below', 'equal', 'above', 'many'])
def test_semch_tile_counts(tiles, prec, monkeypatch):
    """SemCHGraphConv (one mask, 64 channels: one column tile, so tiles = row tiles) and LocalGraph at C = 96 (two
    masks of two column tiles, the second half empty) at tile counts around the SM count; the last row tile is
    partial (J = 17: 7 frames per tile)."""
    import fp64ref as R
    from model.local_attention import LocalGraph, SemCHGraphConv, local_adjacencies
    J, fpt, s = 17, 7, _sms()
    R.install_tables(monkeypatch, J)
    # SemCHGraphConv: tiles = row tiles
    nt = {'below': s - 1, 'equal': s, 'above': s + 1, 'many': 3 * s + 5}[tiles]
    F = fpt * (nt - 1) + 3
    con = local_adjacencies(R.adj(J))[1]
    sc = SemCHGraphConv(64, 64, con, bias=True)
    synth.randomize_module(sc, 80 + nt)
    sc = sc.cuda().eval()
    recs = _audited(sc, _x((1, F, J, 64), nt), prec)
    assert [_tiles(r, fpt) for r in recs] == [nt] and recs[0]['F'] == F
    # LocalGraph, C = 96: 4 column tiles per row tile
    nr = {'below': s // 4 - 1, 'equal': -(-s // 4), 'above': -(-s // 4) + 1, 'many': s + 3}[tiles]
    F = fpt * (nr - 1) + 5
    lg = LocalGraph(R.adj(J), 96, 96, 0.05)
    synth.randomize_module(lg, 90 + nr)
    lg = lg.cuda().eval()
    recs = _audited(lg, _x((1, F, J, 96), nr), prec)
    nt = _tiles(recs[0], fpt)
    assert len(recs) == 1 and nt == 4 * nr
    assert {'below': nt < s, 'equal': s <= nt < s + 4, 'above': s < nt, 'many': nt > 4 * s}[tiles], (nt, s)


PARENTS20 = list(synth.skeleton_parents(19)) + [0]   # the 19-joint skeleton with one more leaf on the root


def _adj(J, monkeypatch):
    """the adjacency of J joints, with the joint table LocalGraph needs (for 20, the leaves are the distal joints)"""
    import fp64ref as R
    import model.local_attention as LA
    if J != 20:
        R.install_tables(monkeypatch, J)
        return R.adj(J)
    from common.graph_utils import adj_mx_from_skeleton
    from common.skeleton import Skeleton
    if J not in LA._JOINT_TABLES:
        monkeypatch.setitem(LA._JOINT_TABLES, 20, ([j for j in range(20) if j not in PARENTS20], [], []))
    return adj_mx_from_skeleton(Skeleton(PARENTS20, [], []))


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
@pytest.mark.parametrize('J', [15, 16, 19, 20])
@pytest.mark.parametrize('C', [32, 64])
def test_semch_joints_and_widths(C, J, prec, monkeypatch):
    """LocalGraph at 8 (J = 15, 16) and 6 (J = 19, 20) frames per tile, about 2.5 tiles per SM, partial last row
    tile."""
    from model.local_attention import LocalGraph
    fpt, s = 128 // J, _sms()
    nr = 5 * s // 4 + 1                              # 2 column tiles per row tile
    F = fpt * (nr - 1) + 1
    lg = LocalGraph(_adj(J, monkeypatch), C, C, 0.05)
    synth.randomize_module(lg, 10 * J + C)
    lg = lg.cuda().eval()
    recs = _audited(lg, _x((1, F, J, C), J + C), prec)
    assert len(recs) == 1 and recs[0]['J'] == J and _tiles(recs[0], fpt) == 2 * nr
