"""GPU: moving live streams between stream pools with their history (PoseStream / GraphedPoseStream .export_streams /
.import_streams, C ABI gast_stream_export / gast_stream_import):
  * the kernels against the numpy model of the state layout (tests/moveref.py), bit for bit, at ring phases from 1 to
    2^40 + phase, into states of another n_streams, J = 17 and 19, first widths 3 and 5, the 81-frame geometry;
  * continuity: pool A runs sequences, exports two streams, pool B of another n imports them at other indices and
    another phase and continues them with the frames A's streams receive; B's poses and indices equal A's bit for bit
    on push_frames / subset calls and GraphedPoseStream ticks (with a peek), and on the single-frame push when the
    phase matches; at another phase the single-frame push stays within the fp64 bars of the stream tests.  Causal and
    not, augment on and off, J = 17 and 19, a first width of 5, the 81-frame geometry at 16 channels, a ring wrap
    between export and import, a stream moved mid-flush, a fresh stream, a round trip through host memory; one case
    on the FFMA core;
  * isolation: an export changes no byte of the source state; an import changes no unlisted stream's snapshot;
  * refusals in C and Python, with both pools' state and counts unchanged, and one launch per move.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from gast_b200 import engine, synth
from gast_b200.realtime import GraphedPoseStream, PoseStream
import delayedref as D
import moveref as M
import streamref as S
import test_gpu_zz_delayed_stream as DS
import test_gpu_zz_stream_exact as X
import test_gpu_zz_subset_stream as SU

pytestmark = pytest.mark.gpu

Case = D.Case
vp = SU.vp
host = SU.host


def geometry(case):
    return case.J, 2, case.fw, case.ch


def move(lib, h, fn, state, n, streams, counts, data, ws=None, nbytes=None):
    s, sp = host(streams, np.int32)
    c, cp = host(counts, np.int64)
    if ws is None:
        ws = torch.empty(int(lib.gast_stream_move_workspace_bytes(h.h, max(1, len(s)))), dtype=torch.uint8,
                         device='cuda')
    return getattr(lib, fn)(h.h, vp(state), n, sp, cp, len(s), vp(data), vp(ws),
                            ws.numel() if nbytes is None else nbytes, C.c_void_p(torch.cuda.current_stream().cuda_stream))


def floats(state):
    """the float view of a state from its 256-byte aligned base (torch allocations are aligned)"""
    assert state.data_ptr() % 256 == 0
    return state.view(torch.float32)


# ---- the kernels against the numpy model --------------------------------------------------------------------------
KCASES = {
    'j17_333_c32': Case(17, (3, 3, 3), 32, 5, 1, 0, (), 61, False, False),
    'j19_333_c16': Case(19, (3, 3, 3), 16, 4, 1, 0, (), 62, True, False),
    'j17_53_c48': Case(17, (5, 3), 48, 6, 1, 0, (), 63, False, False),
    'j17_3333_c16': Case(17, (3, 3, 3, 3), 16, 3, 1, 0, (), 64, False, False),
}


@pytest.mark.parametrize('name', sorted(KCASES))
def test_kernels_equal_numpy_model(name):
    case = KCASES[name]
    m = D.module(case).cuda()
    n, R = case.n, S.receptive_field(case.fw)
    h, lib, st, dev, a = SU.warm_state(case, m, n, R + 4)               # every slot written, rings wrapped
    nf = int(lib.gast_stream_snapshot_floats(h.h))
    assert nf == M.snapshot_floats(*geometry(case))
    src = np.array([n - 1, 0, 1])
    for counts in ([R + 4] * 3, [1, R - 1, X.BIG + 5]):                  # the count only picks the phase
        before = a.clone()
        out = torch.empty((3, nf), device=dev)
        assert move(lib, h, 'gast_stream_export', a, n, src, counts, out) == 0
        assert int(lib.gast_last_launch_count(h.h)) == 1
        assert torch.equal(a, before)
        want = M.export(floats(a).cpu().numpy(), *geometry(case), n, src, counts)
        assert np.array_equal(out.cpu().numpy(), want), counts
        # into a state of n + 2 streams at other indices and phases
        nb = n + 2
        b = torch.from_numpy(np.random.default_rng(1).standard_normal(int(lib.gast_stream_state_bytes(h.h, nb)) // 4)
                             .astype(np.float32)).cuda().view(torch.uint8)
        b0 = floats(b).cpu().numpy()
        dst, cb = np.array([3, nb - 1, 0]), np.array([7, 2 ** 41 + 3, 1])
        assert move(lib, h, 'gast_stream_import', b, nb, dst, cb, out) == 0
        assert int(lib.gast_last_launch_count(h.h)) == 1
        got = floats(b).cpu().numpy()
        assert np.array_equal(got, M.import_(b0, *geometry(case), nb, dst, cb, out.cpu().numpy())), counts


def test_c_refusals():
    case = KCASES['j17_333_c32']
    m = D.module(case).cuda()
    n = case.n
    h, lib, st, dev, state = SU.warm_state(case, m, n, 6)
    nf = int(lib.gast_stream_snapshot_floats(h.h))
    assert lib.gast_stream_move_workspace_bytes(h.h, 0) == 0 and lib.gast_stream_move_workspace_bytes(h.h, 2) > 0
    data = torch.zeros((n + 1, nf), device=dev)
    before, dbefore = state.clone(), data.clone()
    bad = [([0, 0], [6, 6], 'twice'), ([0, 5], [6, 6], 'outside'), ([-1, 1], [6, 6], 'outside'),
           ([0, 1], [6, 0], 'at least 1'), ([], [], 'm must be in'), (list(range(6)), [6] * 6, 'm must be in')]
    for fn in ('gast_stream_export', 'gast_stream_import'):
        for streams, counts, msg in bad:
            assert move(lib, h, fn, state, n, streams, counts, data) != 0, (fn, streams)
            assert msg in engine.L.last_error(), (fn, streams, engine.L.last_error())
        need = int(lib.gast_stream_move_workspace_bytes(h.h, 2))
        ws = torch.empty(need, dtype=torch.uint8, device=dev)
        assert move(lib, h, fn, state, n, [0, 1], [6, 6], data, ws=ws, nbytes=need - 1) != 0
        assert 'workspace too small' in engine.L.last_error()
        assert getattr(lib, fn)(h.h, vp(state), n, vp(None), vp(None), 1, vp(data), vp(ws), need,
                                C.c_void_p(st)) != 0 and 'null' in engine.L.last_error()
        assert move(lib, h, fn, state, 0, [0], [6], data) != 0
    torch.cuda.synchronize()
    assert torch.equal(state, before) and torch.equal(data, dbefore)


# ---- continuity: pool A keeps running, pool B continues the moved streams ------------------------------------------
class Run(object):
    """drives pool A (n_a streams) and pool B (n_b) through the same frames of the moved streams"""

    def __init__(self, case, n_b, mode, K=1, P=0, graphed_src=False):
        self.case, self.mode, self.K, self.P = case, mode, K, P
        self.m = D.module(case).cuda()
        lists = DS.lists(case.J)
        self.lat = D.latency(case.fw, case.causal)

        def pool(n, graphed):
            if graphed:
                return GraphedPoseStream(self.m, n, augment=case.augment, K=K, peek=P, **lists)
            return PoseStream(self.m, n, augment=case.augment, **lists)
        self.A, self.B = pool(case.n, graphed_src), pool(n_b, mode == 'graph')
        self.sa = torch.from_numpy(synth.synth_input(case.n, 1200, case.J, 2, seed=case.seed)).cuda()
        self.sb = torch.from_numpy(synth.synth_input(n_b, 1200, case.J, 2, seed=case.seed + 1)).cuda()
        self.ta = self.tb = 0                        # supply frames used by every stream of A / B

    def tick(self, pool, sel, x):
        """one tick of K frames x (n, K, J, F) on the streams sel -> (poses, index, peek poses, peek index) of sel"""
        sel = list(sel)
        if isinstance(pool, GraphedPoseStream):
            out = pool.push(x, streams=sel)
            return tuple(o[sel] for o in out) + ((None, None) if len(out) == 2 else ())
        if self.mode == 'single':                    # every stream, the lockstep single-frame push
            y, idx = pool.push(x[:, 0])
            return y[sel][:, None], idx[sel][:, None], None, None
        y, idx = pool.push_frames(x[sel].contiguous(), streams=sel)
        py = pidx = None
        if self.P:
            py, pidx = pool.peek(self.P, streams=sel)
        return y, idx, py, pidx

    def run_a(self, ticks, sel=None):
        sel = range(self.case.n) if sel is None else sel
        for _ in range(ticks):
            self.tick(self.A, sel, self.sa[:, self.ta:self.ta + self.K])
            self.ta += self.K

    def run_b(self, ticks):
        for _ in range(ticks):
            self.tick(self.B, range(self.B.n), self.sb[:, self.tb:self.tb + self.K])
            self.tb += self.K

    def both(self, src, dst, ticks, bitwise=True):
        """A ticks on src (every stream in single mode), B on dst with the same frames -> [(pose, key)] of B and A"""
        got = []
        for _ in range(ticks):
            xa = self.sa[:, self.ta:self.ta + self.K]
            xb = self.sb[:, self.tb:self.tb + self.K].clone()
            xb[dst] = xa[src]
            ra = self.tick(self.A, src if self.mode != 'single' else range(self.A.n), xa)
            rb = self.tick(self.B, dst if self.mode != 'single' else range(self.B.n), xb)
            self.ta += self.K
            self.tb += self.K
            if self.mode == 'single':
                ra = tuple(None if r is None else r[src] for r in ra)
                rb = tuple(None if r is None else r[dst] for r in rb)
            ya, ia, pa, pia = ra
            yb, ib, pb, pib = rb
            assert torch.equal(ia, ib)
            due = torch.from_numpy(ia.numpy() >= 0).cuda()
            if bitwise:
                assert torch.equal(ya[due], yb[due])
            if pa is not None:
                assert torch.equal(pia, pib)
                pdue = torch.from_numpy(pia.numpy() >= 0).cuda()
                assert torch.equal(pa[pdue], pb[pdue])
            got.append((yb.cpu().numpy(), ib.numpy()))
        return got

    def flush(self, src, dst, bitwise=True):
        self.A.end(list(src))
        self.B.end(list(dst))
        ticks = -(-self.lat // self.K)
        return self.both(src, dst, ticks, bitwise) if ticks else []


def snapshots_equal(a, b):
    return torch.equal(a.data.view(torch.int32), b.data.view(torch.int32)) and np.array_equal(a.counts, b.counts)


CONT = {
    # case, n_b, mode, K, peek, A ticks, B ticks, moved (src, dst), extras
    'j17_c32_aug_frames_wrap_midflush': (Case(17, (3, 3, 3), 32, 5, 0, 0, (), 71, False, True), 3, 'frames', 3, 0,
                                         14, 40, ([4, 1], [0, 2]), ('midflush',)),
    'j19_c32_causal_frames_fresh': (Case(19, (3, 3, 3), 32, 4, 0, 0, (), 72, True, False), 6, 'frames', 2, 0,
                                    9, 3, ([0, 3], [5, 1]), ('fresh',)),
    'j17_53_c32_aug_frames_host': (Case(17, (5, 3), 32, 3, 0, 0, (), 73, False, True), 2, 'frames', 4, 0,
                                   5, 2, ([2, 0], [1, 0]), ('host',)),
    'j17_3333_c16_aug_frames_peek': (Case(17, (3, 3, 3, 3), 16, 3, 0, 0, (), 74, False, True), 4, 'frames', 5, 7,
                                     20, 1, ([1, 2], [3, 0]), ()),
    'j17_c32_aug_single_phase': (Case(17, (3, 3, 3), 32, 4, 0, 0, (), 75, False, True), 3, 'single', 1, 0,
                                 30, 30 + 27, ([3, 0], [1, 2]), ()),
    'j17_c32_causal_single_phase': (Case(17, (3, 3, 3), 32, 3, 0, 0, (), 76, True, False), 5, 'single', 1, 0,
                                    11, 11 + 2 * 27, ([1, 2], [4, 0]), ()),
    'j17_c32_aug_graph_peek': (Case(17, (3, 3, 3), 32, 5, 0, 0, (), 77, False, True), 3, 'graph', 1, 13,
                               12, 4, ([0, 4], [2, 1]), ('graphed_src', 'midflush')),
    'j19_c16_graph_k2_peek2': (Case(19, (3, 3, 3), 16, 4, 0, 0, (), 78, False, False), 6, 'graph', 2, 2,
                               8, 0, ([3, 1], [0, 5]), ()),
}


def continuity(name, core=0):
    case, n_b, mode, K, P, ta, tb, (src, dst), extras = CONT[name]
    r = Run(case, n_b, mode, K, P, graphed_src='graphed_src' in extras)
    R = S.receptive_field(case.fw)
    r.run_a(ta)
    if 'midflush' in extras:
        r.A.end([src[0]])
        r.run_a(1, sel=src[:1])                      # src[0] has part of its tail pending
        assert r.A.book.left[src[0]] > 0
    if 'fresh' in extras:
        r.A.reset([src[1]])
    r.run_b(tb)
    state_a = r.A._state.clone()
    snap = r.A.export_streams(src)
    assert torch.equal(r.A._state, state_a) and r.A.last_launches == 1
    if 'host' in extras:
        snap = snap.to('cpu')
        assert snap.data.device.type == 'cpu'
    others = [s for s in range(n_b) if s not in dst]
    keep = r.B.export_streams(others) if others else None
    counts_b = r.B.counts.copy()
    r.B.import_streams(snap, dst)
    assert r.B.last_launches == 1
    assert not others or snapshots_equal(r.B.export_streams(others), keep)
    assert np.array_equal(np.delete(r.B.counts, dst), np.delete(counts_b, dst))
    assert (r.B.counts[dst] == max(counts_b.min(), 1)).all()
    if mode == 'single':
        assert (r.A.step - r.B.step) % R == 0 and not r.B._delta.any()
    if mode == 'graph':
        g = r.B
        assert np.array_equal(g._counts_dev.view(g.copies, n_b).cpu().numpy(), np.tile(g.counts, (g.copies, 1)))
    r.both(src, dst, R + 3)                          # more than a ring wrap after the import
    r.flush(src, dst)
    DS.report('move %s core %d: bitwise over %d ticks' % (name, core, R + 3))


@pytest.mark.parametrize('name', sorted(CONT))
def test_moved_streams_continue_bitwise(name):
    continuity(name)


def test_moved_streams_continue_bitwise_ffma():
    engine.set_gemm_core(1)
    try:
        continuity('j17_c32_aug_frames_wrap_midflush', core=1)
    finally:
        engine.set_gemm_core(0)


@pytest.mark.parametrize('causal', [False, True])
def test_single_push_at_another_phase_vs_fp64(causal):
    """B's lockstep single-frame push at another phase than A's: the poses of the moved streams' sequences against
    the fp64 poses of those sequences (the stream tests' bars); the indices equal A's"""
    case = Case(17, (3, 3, 3), 32, 4, 0, 0, (), 79, causal, True)
    r = Run(case, 3, 'single')
    src, dst = [2, 0], [1, 2]
    r.run_a(17)
    r.run_b(17 + 5)
    r.B.import_streams(r.A.export_streams(src), dst)
    assert (r.A.step - r.B.step) % S.receptive_field(case.fw) != 0
    got = r.both(src, dst, 40, bitwise=False) + r.flush(src, dst, bitwise=False)
    seqs = [r.sa[s, :17 + 40].cpu().numpy() for s in src]
    ref = D.sequence_poses(seqs, case.J, case.fw, case.causal, True, D.symmetry(case.J), D.module(case).state_dict())
    a, b = [], []
    for y, idx in got:
        for i in range(2):
            for k in np.flatnonzero(idx[i] >= 0):
                a.append(y[i, k])
                b.append(ref[i][idx[i, k]])
    assert len(a) == 2 * (40 + r.lat)
    mx, l2 = S.errors(np.stack(a), np.stack(b))
    DS.report('move single-frame push at another phase causal %d: max %.2e l2 %.2e' % (causal, mx, l2))
    assert mx <= X.MAX_BAR and l2 <= X.L2_BAR, (mx, l2)


# ---- refusals -----------------------------------------------------------------------------------------------------
def pool_state(p):
    return (None if p._state is None else p._state.clone(), p.counts.copy(), p.book.rows(range(p.n)))


def same_state(p, s):
    st, counts, rows = s
    return ((st is None and p._state is None) or torch.equal(p._state, st)) and np.array_equal(p.counts, counts) and \
        all(np.array_equal(x, y) for x, y in zip(p.book.rows(range(p.n)), rows))


def test_python_refusals():
    case = Case(17, (3, 3, 3), 32, 4, 0, 0, (), 81, False, True)
    m = D.module(case).cuda()
    x = torch.from_numpy(synth.synth_input(4, 20, 17, 2, seed=3)).cuda()
    a, b = PoseStream(m, 4, augment=True), PoseStream(m, 3, augment=True)
    a.push_frames(x[:, :6])
    b.push_frames(x[:3, 6:9])
    snap = a.export_streams([1, 2])
    sa, sb = pool_state(a), pool_state(b)
    other = D.module(case._replace(seed=82)).cuda()
    wide = D.module(case._replace(ch=64)).cuda()
    refusals = [
        (PoseStream(wide, 3, augment=True), snap, [0, 1], 'architecture'),
        (PoseStream(m, 3), snap, [0, 1], 'augment'),
        (PoseStream(m, 3, augment=True, joints_left=[1, 2, 3, 14, 15, 16], joints_right=[4, 5, 6, 11, 12, 13]), snap,
         [0, 1], 'symmetry'),
        (PoseStream(other, 3, augment=True), snap, [0, 1], 'another model object'),
        (b, snap, [0], 'listed'),
        (b, snap, [0, 0], 'streams'),
        (b, snap, [0, 3], 'streams'),
        (b, 'not a snapshot', [0, 1], 'StreamSnapshot'),
    ]
    for pool, s, streams, msg in refusals:
        with pytest.raises(engine.GastError, match=msg):
            pool.import_streams(s, streams)
    with pytest.raises(engine.GastError, match='streams'):
        a.export_streams([1, 1])
    with pytest.raises(engine.GastError, match='streams'):
        a.export_streams([4])
    assert same_state(a, sa) and same_state(b, sb)
    # the weights change after the export: the snapshot is refused, and the source refuses to export
    X._change('load_state_dict', m, S.Case(17, (3, 3, 3), 32, 4, 30, 0, (), 83))
    with pytest.raises(engine.GastError, match='since the export'):
        b.import_streams(snap, [0, 1])
    with pytest.raises(engine.GastError, match='reset'):
        a.export_streams([0])
    assert same_state(a, sa) and same_state(b, sb)
    # a precision or GEMM-core switch is not a weight change
    m2 = D.module(case).cuda()
    c, d = PoseStream(m2, 2, augment=True), PoseStream(m2, 2, augment=True)
    c.push_frames(x[:2, :5])
    engine.set_precision(m2, 'tf32')
    try:
        d.import_streams(c.export_streams([0]), [1])
    finally:
        engine.set_precision(m2, 'fp32')
    engine.set_gemm_core(1)
    try:
        d.import_streams(c.export_streams([1]), [0])
    finally:
        engine.set_gemm_core(0)
    assert d.counts.tolist() == [1, 1] and not d.book.fresh.any()


def test_graphed_pool_refusals_keep_counts():
    case = Case(17, (3, 3, 3), 32, 3, 0, 0, (), 84, False, False)
    m = D.module(case).cuda()
    g = GraphedPoseStream(m, 3, peek=2)
    e = PoseStream(m, 2)
    x = torch.from_numpy(synth.synth_input(3, 10, 17, 2, seed=4)).cuda()
    for t in range(4):
        g.push(x[:, t:t + 1])
    snap = e.export_streams([0, 1])                  # never pushed: fresh streams
    sg, dev_counts = pool_state(g), g._counts_dev.clone()
    with pytest.raises(engine.GastError, match='listed'):
        g.import_streams(snap, [0])
    with pytest.raises(engine.GastError, match='streams'):
        g.import_streams(snap, [2, 2])
    assert same_state(g, sg) and torch.equal(g._counts_dev, dev_counts)
    graph = g.graph
    g.import_streams(snap, [2, 0])                   # fresh streams stay fresh, at count step = 4
    assert g.graph is graph and g.book.fresh.tolist() == [True, False, True]
    assert g._counts_dev.tolist() == [4, 4, 4] and g.counts.tolist() == [4, 4, 4]
