"""GPU: stream ticks driven by frame counts on the device (C ABI gast_stream_push_device / gast_stream_peek_device) and
replayed from a CUDA graph (GraphedPoseStream), on both GEMM cores:
  * the device entries against the subset entries on the seeded schedules of the subset-stream file (resets, ends,
    a stream sitting out more than R_max ticks, ring wraps, sequences shorter than the latency, counts from
    2^40 + phase, K varying between calls): every active row, the whole state byte for byte and the counts;
  * inactive streams: NaN rows of x change no active bit and no byte of an inactive stream's state;
  * a count of 0 is a fresh stream, a negative count is 0;
  * GraphedPoseStream ticks bitwise those of a PoseStream driven by the same `streams=` calls (poses, peek poses,
    indices), causal and not, augment on and off, J = 17 and 19, K = 1 and K > 1; one case against fp64 (TF32 on
    one more); the two-person demo case against tta.evaluate_sequence;
  * refusals in C and in Python, the recapture after a weight change with every stream reset, and launch counts.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from gast_b200 import engine, synth, tta
from gast_b200.realtime import GraphedPoseStream, PoseStream, SequenceBook
import delayedref as D
import streamref as S
import test_gpu_zz_delayed_stream as DS
import test_gpu_zz_stream_exact as X
import test_gpu_zz_subset_stream as SU

pytestmark = pytest.mark.gpu

Case = D.Case
CASES = DS.CASES
vp = SU.vp


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def dev_i32(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).cuda()


def push_device(lib, h, state, n, counts, active, K, x, y, ws, st, fresh=None, hold=None, nbytes=None):
    return lib.gast_stream_push_device(h.h, vp(state), n, vp(counts), vp(active), K, vp(x), vp(y), vp(fresh),
                                       vp(hold), vp(ws), ws.numel() if nbytes is None else nbytes, C.c_void_p(st))


def peek_device(lib, h, state, n, counts, active, K, y, ws, st, nbytes=None):
    return lib.gast_stream_peek_device(h.h, vp(state), n, vp(counts), vp(active), K, vp(y), vp(ws),
                                       ws.numel() if nbytes is None else nbytes, C.c_void_p(st))


# ---- the C entries against the subset entries --------------------------------------------------------------------
@pytest.mark.parametrize('name', sorted(CASES))
def test_device_entries_equal_subset_entries(name, core, plans):
    case = CASES[name]
    calls, _, supply, _ = SU.get_plan(plans, name)
    m = D.module(case).cuda()
    h, lib, st, dev = SU.abi(m)
    n, J, lat = case.n, case.J, D.latency(case.fw, case.causal)
    nb = int(lib.gast_stream_state_bytes(h.h, n))
    a = torch.zeros(nb, dtype=torch.uint8, device=dev)      # the subset entries' state
    b = a.clone()                                            # the device entries' state
    kmax = max(K for _, _, K, *_ in calls)
    wa = torch.empty(int(lib.gast_stream_subset_workspace_bytes(h.h, n, max(kmax, lat))), dtype=torch.uint8,
                     device=dev)
    wb = torch.empty(int(lib.gast_stream_device_workspace_bytes(h.h, n, max(kmax, lat))), dtype=torch.uint8,
                     device=dev)
    counts = np.full(n, case.start, dtype=np.int64)
    dcounts = torch.from_numpy(counts.copy()).cuda()
    book = SequenceBook(n, lat)
    rng = np.random.default_rng(case.seed)
    for q, (events, sel, K, valid, src, index, _) in enumerate(calls):
        for kind, ss in events:
            getattr(book, kind)(ss)
        fresh, hold, _ = book.advance_many(K, valid, streams=sel)
        x = torch.from_numpy(synth.synth_input(n, K, J, 2, seed=q)).cuda()
        on = np.zeros(n, dtype=bool)
        on[sel] = True
        x[torch.from_numpy(~on).cuda()] = float('nan')      # never read
        fr, ho = np.zeros(n, dtype=np.int32), np.zeros((n, K), dtype=np.int32)
        fr[sel], ho[sel] = fresh, hold
        ya = torch.empty((sel.size, K, J, 3), device=dev)
        yb = torch.full((n, K, J, 3), float('nan'), device=dev)
        selt = torch.from_numpy(sel).cuda()
        # a stream at count 0 must be fresh for the subset entry (one ended before its first frame is not); the
        # device entry makes it fresh itself
        assert SU.push_subset(lib, h, a, n, sel, counts[sel], K, x[selt].contiguous(), ya, wa, st,
                              fresh=dev_i32(fresh | (counts[sel] == 0)), hold=dev_i32(hold)) == 0
        active = None if on.all() and q % 2 else dev_i32(on)
        assert push_device(lib, h, b, n, dcounts, active, K, x, yb, wb, st, fresh=dev_i32(fr), hold=dev_i32(ho)) == 0
        counts[sel] += K
        assert torch.equal(yb[selt], ya) and not torch.isnan(ya).any(), (name, q)
        assert torch.equal(a, b), (name, q)
        assert np.array_equal(dcounts.cpu().numpy(), counts), (name, q)
        if lat and q % 3 == 0:
            P = int(rng.integers(1, lat + 1))
            pick = sel[counts[sel] >= 1]
            pa = torch.empty((pick.size, P, J, 3), device=dev)
            pb = torch.empty((n, P, J, 3), device=dev)
            assert SU.peek_subset(lib, h, a, n, pick, counts[pick], P, pa, wa, st) == 0
            assert peek_device(lib, h, b, n, dcounts, dev_i32(on), P, pb, wb, st) == 0
            assert torch.equal(pb[torch.from_numpy(pick).cuda()], pa), (name, q)
    assert torch.equal(a, b) and np.array_equal(dcounts.cpu().numpy(), counts)


@pytest.fixture(scope='module')
def plans():
    return {}


def test_inactive_streams_are_isolated(core):
    """NaN rows of the inactive streams: the active rows are bitwise those of an all-finite call and hold no NaN, and
    no byte of an inactive stream's state changes"""
    case = Case(16, (3, 5, 3), 32, 7, 1, 0, (), 85, False, False)
    m = D.module(case).cuda()
    n, J = case.n, case.J
    h, lib, st, dev, base = SU.warm_state(case, m, n, 12)
    ws = torch.empty(int(lib.gast_stream_device_workspace_bytes(h.h, n, 40)), dtype=torch.uint8, device=dev)
    on = np.array([0, 1, 0, 1, 1, 0, 0], dtype=bool)
    act = torch.from_numpy(on).cuda()
    before = SU.state_rows(case, base, n)
    for K in (1, 40):                        # 40 frames: more than a ring of 15 slots, every slot rewritten
        s1, s2 = base.clone(), base.clone()
        c1 = torch.full((n,), 12, dtype=torch.int64, device=dev)
        c2 = c1.clone()
        x = torch.from_numpy(synth.synth_input(n, K, J, 2, seed=K)).cuda()
        y1, y2 = torch.empty((n, K, J, 3), device=dev), torch.empty((n, K, J, 3), device=dev)
        assert push_device(lib, h, s1, n, c1, dev_i32(on), K, x, y1, ws, st) == 0
        xn = x.clone()
        xn[~act] = float('nan')
        assert push_device(lib, h, s2, n, c2, dev_i32(on), K, xn, y2, ws, st) == 0
        assert torch.equal(y1[act], y2[act]) and torch.isfinite(y2[act]).all()
        assert torch.equal(s1, s2) and torch.equal(c1, c2)
        after = SU.state_rows(case, s2, n)
        for s in range(n):
            assert torch.equal(before[s], after[s]) == (not on[s]), (K, s)
        assert c1.tolist() == [12 + K * int(o) for o in on]


def test_count_zero_is_fresh_and_negative_is_zero(core):
    case = Case(17, (3, 3, 3), 32, 5, 1, 0, (), 83, False, True)
    m = D.module(case).cuda()
    n, J, K = case.n, case.J, 3
    h, lib, st, dev, state = SU.warm_state(case, m, n, 20)
    ws = torch.empty(int(lib.gast_stream_device_workspace_bytes(h.h, n, K)), dtype=torch.uint8, device=dev)
    x = torch.from_numpy(synth.synth_input(n, K, J, 2, seed=4)).cuda()
    outs = []
    for start, fresh in ((0, np.ones(n)), (0, None), (-5, None), (-(2 ** 62), np.ones(n))):
        s = state.clone()
        c = torch.full((n,), start, dtype=torch.int64, device=dev)
        y = torch.empty((n, K, J, 3), device=dev)
        assert push_device(lib, h, s, n, c, None, K, x, y, ws, st, fresh=None if fresh is None else dev_i32(fresh)) == 0
        assert c.tolist() == [K] * n
        outs.append((y, s))
    for y, s in outs[1:]:
        assert torch.equal(y, outs[0][0]) and torch.equal(s, outs[0][1])
    # a peek at count 0 reads no ring and faults on nothing; the streams with a count are the subset peek's
    c = torch.tensor([0, 20, -3, 2 ** 62, 20], dtype=torch.int64, device=dev)
    pw = torch.empty(int(lib.gast_stream_device_workspace_bytes(h.h, n, 13)), dtype=torch.uint8, device=dev)
    yp = torch.empty((n, 13, J, 3), device=dev)
    before = state.clone()
    assert peek_device(lib, h, state, n, c, None, 13, yp, pw, st) == 0
    assert torch.equal(state, before) and c.tolist() == [0, 20, -3, 2 ** 62, 20]
    ya = torch.empty((2, 13, J, 3), device=dev)
    sw = torch.empty(int(lib.gast_stream_subset_workspace_bytes(h.h, 2, 13)), dtype=torch.uint8, device=dev)
    assert SU.peek_subset(lib, h, state, n, [1, 4], [20, 20], 13, ya, sw, st) == 0
    assert torch.equal(yp[[1, 4]], ya)


# ---- GraphedPoseStream against PoseStream --------------------------------------------------------------------------
GCASES = {
    # J, fw, channels, n streams, causal, augment, K, peek (-1: latency)
    'j17_c32_n5_aug_k1_peek': (17, (3, 3, 3), 32, 5, False, True, 1, -1),
    'j19_c32_n4_k3_peek2': (19, (3, 3, 3), 32, 4, False, False, 3, 2),
    'j17_c64_causal_n3_aug_k2': (17, (3, 3, 3), 64, 3, True, True, 2, 0),
    'j19_c16_causal_n6_k1': (19, (3, 3, 3), 16, 6, True, False, 1, 0),
    'j17_c32_n6_k4': (17, (3, 3, 3), 32, 6, False, False, 4, 0),
}


def gcase(name, seed=0):
    J, fw, ch, n, causal, aug, K, P = GCASES[name]
    case = Case(J, fw, ch, n, 1, 0, (), 300 + seed, causal, aug)
    return case, K, (D.latency(fw, causal) if P < 0 else P)


def schedule(n, lat, ticks, seed):
    """[(events, sel or None)]: every tick changes the active set and, most ticks, resets or ends a stream"""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(ticks):
        events = []
        if t and rng.random() < 0.4:
            events.append(('reset', [int(rng.integers(n))]))
        if t and rng.random() < 0.4:
            events.append(('end', [int(rng.integers(n))]))
        if t % 7 == 0:
            sel = None
        else:
            sel = sorted(int(s) for s in rng.permutation(n)[:int(rng.integers(1, n + 1))])
            if rng.random() < 0.5:
                sel = sel[::-1]
        out.append((events, sel))
    return out


def run_both(model, case, K, P, ticks, seed):
    """tick a GraphedPoseStream and a PoseStream through one schedule, every tick checked bitwise (the rows with a
    pose due) -> the graphed stream"""
    n, lat = case.n, D.latency(case.fw, case.causal)
    lists = DS.lists(case.J)
    g = GraphedPoseStream(model, n, augment=case.augment, K=K, peek=P, **lists)
    e = PoseStream(model, n, augment=case.augment, **lists)
    supply = torch.from_numpy(synth.synth_input(n, ticks * K + 1, case.J, 2, seed=seed)).cuda()
    for t, (events, sel) in enumerate(schedule(n, lat, ticks, seed)):
        for kind, ss in events:
            getattr(g, kind)(ss)
            getattr(e, kind)(ss)
        rows = list(range(n)) if sel is None else sel
        frames = supply[:, t * K:(t + 1) * K].clone()
        got = g.push(frames, streams=sel)
        ye, ie = e.push_frames(frames[rows].contiguous(), streams=rows)
        idx = got[1].numpy()
        assert np.array_equal(idx[rows], ie.numpy()) and (np.delete(idx, rows, 0) == -1).all(), t
        due = torch.from_numpy(ie.numpy() >= 0).cuda()
        assert torch.equal(got[0][rows][due], ye[due]), t
        if P:
            pe, pie = e.peek(P, streams=rows)
            assert np.array_equal(got[3].numpy()[rows], pie.numpy()), t
            pdue = torch.from_numpy(pie.numpy() >= 0).cuda()
            assert torch.equal(got[2][rows][pdue], pe[pdue]), t
        assert np.array_equal(g.counts, e.counts), t
    assert np.array_equal(g._counts_dev.view(g.copies, n).cpu().numpy(), np.tile(g.counts, (g.copies, 1)))
    return g


@pytest.mark.parametrize('name', sorted(GCASES))
def test_graph_ticks_equal_pose_stream(name, core):
    case, K, P = gcase(name)
    ticks = 3 * SU.r_max(case.fw) + 5
    run_both(D.module(case).cuda(), case, K, P, ticks, seed=len(name))


def test_graph_ticks_vs_fp64():
    """one non-causal augmented case, every returned pose against the fp64 poses of the sequences each stream
    received (the subset file's bars), then the same in TF32"""
    case, K, P = gcase('j17_c32_n5_aug_k1_peek')
    for prec, bar in (('fp32', None), ('tf32', SU.TF32_BAR)):
        m = engine.set_precision(D.module(case).cuda(), prec)
        n, lat = case.n, D.latency(case.fw, case.causal)
        g = GraphedPoseStream(m, n, augment=True, K=1)
        supply = synth.synth_input(n, 200, case.J, 2, seed=77)
        seqs = [[] for _ in range(n)]            # frames of each stream's sequences
        got = {}
        sched = schedule(n, lat, 3 * SU.r_max(case.fw), 5)
        sched.append(([('end', None)], None))
        sched += [([], None)] * lat
        for events, sel in sched:
            for kind, ss in events:
                getattr(g, kind)(ss)
            rows = list(range(n)) if sel is None else sel
            starting = g.book.fresh.copy()
            live = g.book.left < 0
            frames = np.full((n, 1, case.J, 2), np.nan, dtype=np.float32)
            for s in rows:
                if starting[s]:
                    seqs[s].append([])
                if starting[s] or live[s]:
                    f = supply[s, sum(len(q) for q in seqs[s])]
                    seqs[s][-1].append(f)
                    frames[s, 0] = f
            y, idx = g.push(torch.from_numpy(frames).cuda(), streams=sel)
            for s in rows:
                if idx[s, 0] >= 0:
                    got[(s, len(seqs[s]) - 1, int(idx[s, 0]))] = y[s, 0].cpu().numpy()
        keys = sorted(got)
        qs = sorted({(s, k) for s, k, _ in keys})
        ref = D.sequence_poses([np.stack(seqs[s][k]) for s, k in qs], case.J, case.fw, case.causal, True,
                               D.symmetry(case.J), D.module(case).state_dict())
        ref = dict(zip(qs, ref))
        a = np.stack([got[k] for k in keys])
        b = np.stack([ref[(s, k)][j] for s, k, j in keys])
        mx, l2 = S.errors(a, b)
        DS.report('graph %s: max %.2e l2 %.2e | %d poses' % (prec, mx, l2, len(keys)))
        if bar is None:
            assert mx <= SU.MAX_BAR and l2 <= SU.L2_BAR, (mx, l2)
        else:
            assert mx < bar, mx


def test_two_persons_with_different_valid_frames(core):
    """the reference's num_person = 2 demo: each person active on its own valid frames only equals
    tta.evaluate_sequence of that person's valid frames"""
    case = Case(17, (3, 3, 3), 128, 2, 90, 0, (), 91, False, True)
    m = D.module(case, dilated=True).cuda()
    kpts = D.frames(case)
    valid = [np.ones(case.T, dtype=bool), np.ones(case.T, dtype=bool)]
    valid[1][20:36] = False
    valid[1][60:71] = False
    valid[0][:3] = False
    g = GraphedPoseStream(m, 2, augment=True)
    x = torch.from_numpy(kpts).cuda()
    got = [[], []]

    def tick(frames, sel):
        y, idx = g.push(frames, streams=sel)
        for p in sel:
            if idx[p, 0] >= 0:
                assert idx[p, 0] == len(got[p])
                got[p].append(y[p, 0].clone())
    for t in range(case.T):
        tick(x[t][:, None], [p for p in (0, 1) if valid[p][t]])
    g.end()
    for _ in range(g.latency):
        tick(torch.full((2, 1, 17, 2), float('nan')), [0, 1])
    kl, kr, jl, jr = D.symmetry(17)
    for p in (0, 1):
        want = tta.evaluate_sequence(m, kpts[valid[p], p], kl, kr, jl, jr, causal=False).cpu().numpy()
        gp = torch.stack(got[p]).cpu().numpy()
        assert gp.shape == want.shape, (p, gp.shape)
        w = float(np.abs(gp - want).max() / np.abs(want).max())
        DS.report('graph two persons core %d person %d: %.2e' % (core, p, w))
        assert w <= DS.WHOLE_BAR, w


# ---- refusals, recapture, launch counts ----------------------------------------------------------------------------
def test_c_refusals():
    case = Case(17, (3, 3, 3), 32, 4, 1, 0, (), 95, False, False)
    m = D.module(case).cuda()
    h, lib, st, dev, state = SU.warm_state(case, m, 4, 6)
    n, K, J = 4, 3, 17
    wb = int(lib.gast_stream_device_workspace_bytes(h.h, n, 13))
    assert wb > 0 and lib.gast_stream_device_workspace_bytes(h.h, 0, K) == 0
    assert lib.gast_stream_device_workspace_bytes(h.h, n, 0) == 0
    ws = torch.empty(wb, dtype=torch.uint8, device=dev)
    x = torch.zeros((n, K, J, 2), device=dev)
    y = torch.empty((n, 13, J, 3), device=dev)
    c = torch.full((n,), 6, dtype=torch.int64, device=dev)
    before = state.clone()
    assert push_device(lib, h, state, n, None, None, K, x, y, ws, st) != 0 and 'null counts' in engine.L.last_error()
    assert peek_device(lib, h, state, n, None, None, 1, y, ws, st) != 0 and 'null counts' in engine.L.last_error()
    assert push_device(lib, h, state, n, c, None, 0, x, y, ws, st) != 0 and 'K must be' in engine.L.last_error()
    assert push_device(lib, h, state, 0, c, None, K, x, y, ws, st) != 0
    for P in (0, 14):
        assert peek_device(lib, h, state, n, c, None, P, y, ws, st) != 0
        assert 'K must be in [1, latency = 13]' in engine.L.last_error()
    need = int(lib.gast_stream_device_workspace_bytes(h.h, n, K))
    assert push_device(lib, h, state, n, c, None, K, x, y, ws, st, nbytes=need - 1) != 0
    assert 'workspace too small' in engine.L.last_error()
    assert torch.equal(state, before) and c.tolist() == [6] * n
    hc = SU.abi(D.module(case._replace(causal=True)).cuda())[0]
    assert peek_device(lib, hc, state, n, c, None, 1, y, ws, st) != 0 and 'non-causal' in engine.L.last_error()
    from model.gast_net import SpatioTemporalModel
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    dense = SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], channels=16, dense=True).cuda().eval()
    hd = SU.abi(dense)[0]
    assert push_device(lib, hd, state, n, c, None, K, x, y, ws, st) != 0 and 'dense' in engine.L.last_error()
    assert torch.equal(state, before) and c.tolist() == [6] * n
    assert push_device(lib, h, state, n, c, None, K, x, y, ws, st) == 0 and c.tolist() == [9] * n


def test_python_refusals_and_recapture():
    case = Case(17, (3, 3, 3), 32, 4, 1, 0, (), 97, False, True)
    m = D.module(case).cuda()
    n, J = case.n, case.J
    with pytest.raises(engine.GastError, match='peek'):
        GraphedPoseStream(m, n, peek=14)
    with pytest.raises(engine.GastError, match='K must'):
        GraphedPoseStream(m, n, K=0)
    g = GraphedPoseStream(m, n, augment=True, peek=2)
    x = torch.from_numpy(synth.synth_input(n, 40, J, 2, seed=8)).cuda()
    for t in range(5):
        g.push(x[:, t:t + 1])
    graph = g.graph
    with pytest.raises(engine.GastError):
        g.push_frames(x[:, :1])
    with pytest.raises(engine.GastError, match='streams'):
        g.push(x[:, :1], streams=[0, 0])
    m.train()
    with pytest.raises(engine.GastError, match='eval'):
        g.push(x[:, 5:6])
    m.eval()
    engine.set_precision(m, 'tf32')
    with pytest.raises(engine.GastError, match='set_precision'):
        g.push(x[:, 5:6])
    engine.set_precision(m, 'fp32')
    engine.set_gemm_core(1)
    try:
        with pytest.raises(engine.GastError, match='set_gemm_core'):
            g.push(x[:, 5:6])
    finally:
        engine.set_gemm_core(0)
    assert g.counts.tolist() == [5] * n and g.graph is graph
    X._change('load_state_dict', m, S.Case(17, (3, 3, 3), 32, 4, 30, 0, (), 98))
    with pytest.raises(engine.GastError, match='reset'):
        g.push(x[:, 5:6])
    g.reset([0, 1])
    with pytest.raises(engine.GastError, match='reset'):
        g.push(x[:, 5:6])
    assert g.counts.tolist() == [5] * n
    g.reset()
    e = PoseStream(m, n, augment=True)
    e.step = 5
    for t in range(5, 12):
        y, idx, py, pidx = g.push(x[:, t:t + 1])
        ye, ie = e.push_frames(x[:, t:t + 1])
        pe, pie = e.peek(2)
        assert torch.equal(idx, ie) and torch.equal(pidx, pie)
        due, pdue = torch.from_numpy(ie.numpy() >= 0).cuda(), torch.from_numpy(pie.numpy() >= 0).cuda()
        assert torch.equal(y[due], ye[due]) and torch.equal(py[pdue], pe[pdue]), t
    assert g.graph is not graph


def test_launch_counts():
    case = Case(17, (3, 3, 3), 64, 1, 1, 0, (), 9, False, False)
    m = D.module(case).cuda()
    J = case.J
    counts = set()
    for n in (3, 40):
        h, lib, st, dev, state = SU.warm_state(case, m, n, 5)
        for K in (1, 6):
            ws = torch.empty(int(lib.gast_stream_device_workspace_bytes(h.h, n, 13)), dtype=torch.uint8, device=dev)
            cw = torch.empty(int(lib.gast_stream_chunk_workspace_bytes(h.h, n, 13)), dtype=torch.uint8, device=dev)
            x = torch.zeros((n, K, J, 2), device=dev)
            y = torch.empty((n, 13, J, 3), device=dev)
            assert lib.gast_stream_push_chunk(h.h, vp(state.clone()), C.c_int64(5), vp(x), vp(y), n, K, vp(None),
                                              vp(None), vp(cw), cw.numel(), C.c_void_p(st)) == 0
            chunk = int(lib.gast_last_launch_count(h.h))
            assert lib.gast_stream_peek(h.h, vp(state), C.c_int64(5), vp(y), n, min(K, 13), vp(cw), cw.numel(),
                                        C.c_void_p(st)) == 0
            peek = int(lib.gast_last_launch_count(h.h))
            for on in (None, np.ones(n), np.eye(n)[1], np.zeros(n)):
                c = torch.full((n,), 5, dtype=torch.int64, device=dev)
                act = None if on is None else dev_i32(on)
                assert push_device(lib, h, state.clone(), n, c, act, K, x, y, ws, st) == 0
                assert int(lib.gast_last_launch_count(h.h)) == chunk + 1
                assert peek_device(lib, h, state, n, c, act, min(K, 13), y, ws, st) == 0
                assert int(lib.gast_last_launch_count(h.h)) == peek + 1
            counts.add((chunk, peek))
    assert len(counts) == 1, counts
    chunk, peek = counts.pop()
    g = GraphedPoseStream(m, 4, augment=True, peek=13)
    g.push(torch.zeros(4, 1, J, 2))
    assert g.last_launches == (chunk + 1) + (peek + 1) + 3        # gast_tta_prepare and two gast_tta_merge
