"""GPU: any subset of the streams, each at its own frame count (PoseStream.push / push_frames / peek with `streams`,
C ABI gast_stream_push_subset / gast_stream_peek_subset), on both GEMM cores:
  * seeded random schedules over the geometries of the delayed-stream matrix (tests/test_gpu_zz_delayed_stream.py):
    ticks of one stream, of every stream and of random subsets pushing K = 1, 2, 5, 7 frames, resets and ends of single
    streams, a stream left untouched for more than R_max ticks while the others wrap their rings several times, an end
    on a stream's own ring wrap, a sequence shorter than the latency, counts from 2^40 + phase, the final flush; every
    returned pose of the sampled streams against the fp64 poses of the sequences those streams received (TF32 on one
    case);
  * bitwise: a subset of every stream at one step against gast_stream_push_chunk (in order and reversed), peek_subset
    against gast_stream_peek, the bytes of unlisted streams and of the whole state after a peek;
  * PoseStream: calls without `streams` bitwise those of a stream that never used subsets, peeks after the phases
    diverged against a held push of a clone, with the index of the book;
  * two persons with different valid frames (the reference's gen_pose for num_person = 2) against
    tta.evaluate_sequence of each person's valid frames;
  * refusals in C and Python, and launch counts that depend on neither n, m nor K.

Measured on an H100 80GB HBM3 (700 W power limit), worst over the schedules and both GEMM cores, against fp64: max
error / max |y64| 2.8e-6 (the 243-frame model; 1.6e-6 at most elsewhere), relative L2 1.7e-6; TF32 9.2e-4; the two
persons equal evaluate_sequence bit for bit.  The bars are the delayed-stream file's (about 3-4x those; TF32 that of
the peek file).  The file runs in about 40 s.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from gast_b200 import engine, synth, tta
from gast_b200.realtime import CausalStream, PoseStream, SequenceBook
import delayedref as D
import streamref as S
import test_gpu_zz_delayed_stream as DS
import test_gpu_zz_stream_exact as X

pytestmark = pytest.mark.gpu

MAX_BAR = DS.MAX_BAR
L2_BAR = DS.L2_BAR
TF32_BAR = 5e-3                    # max |y - y64| / max |y64| in TF32 (DESIGN.md §4.1)
Case = D.Case
CASES = DS.CASES


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def r_max(fw):
    return S.receptive_field(fw)


# ---- random schedules --------------------------------------------------------------------------------------------
SLEEPER, WRAPPER, SHORT = 0, 1, 2           # the stream left untouched, the one ended on its ring wrap, the short one


def plan(case):
    """A seeded schedule of subset calls, built on a host SequenceBook.  -> (calls, seqs, cut) with
    calls = [(events [(kind, [s])], sel, K, valid or None, src (m,) first supply frame, index (m, K), seq (m,))],
    seqs[s] = [(first supply frame, length)] of every sequence stream s received (supply frames are consumed in order)
    and cut = the streams whose last sequence a reset cut short before the final flush.  Random events touch the
    streams after SHORT only."""
    rng = np.random.default_rng(1000 + case.seed)
    n, R, lat = case.n, r_max(case.fw), D.latency(case.fw, case.causal)
    book = SequenceBook(n, lat)
    count = np.full(n, case.start, dtype=np.int64)
    used = np.zeros(n, dtype=np.int64)
    seqs = [[] for _ in range(n)]
    calls = []
    sleep = range(8, 8 + 2 * R)                # SLEEPER sits out 2 R_max ticks
    ticks = 8 + 2 * R + 20

    def call(events, sel, K, valid=None):
        for kind, ss in events:
            getattr(book, kind)(ss)
        sel = np.asarray(sel, dtype=np.int64)
        starting = book.fresh[sel].copy()
        fresh, hold, index = book.advance_many(K, valid, streams=sel)
        src, seq = np.zeros(sel.size, dtype=np.int64), np.zeros(sel.size, dtype=np.int64)
        for i, s in enumerate(sel):
            if starting[i]:
                seqs[s].append([int(used[s]), 0])
            take = int((~hold[i]).sum())
            src[i] = used[s]
            used[s] += take
            if seqs[s]:
                seqs[s][-1][1] += take
            seq[i] = len(seqs[s]) - 1
        count[sel] += K
        calls.append((events, sel, K, valid, src, index, seq))

    for t in range(ticks):
        events = []
        if n > 3 and t > 0 and rng.random() < 0.2:
            events.append(('reset', [int(rng.integers(3, n))]))
        if n > 3 and t > 0 and rng.random() < 0.2:
            events.append(('end', [int(rng.integers(3, n))]))
        idle = np.flatnonzero((book.left == 0) & ~book.fresh)
        if idle.size and rng.random() < 0.5:     # an ended stream (by valid or an event) restarts
            events.append(('reset', [int(rng.choice(idle))]))
        if t == 20:                                # WRAPPER alone up to its own ring wrap, then its end
            call(events, [WRAPPER], int(-count[WRAPPER] % R) or R)
            events = [('end', [WRAPPER])]
        if t == 24:
            events.append(('reset', [WRAPPER]))
        if t == 30:                                # SHORT: a sequence of 2 frames (< latency), then more of it held
            call(events + [('reset', [SHORT])], [SHORT], 2)
            events = [('end', [SHORT])]
        if t == 40:
            events.append(('reset', [SHORT]))
        pool = [s for s in range(n) if not (t in sleep and s == SLEEPER)]
        kind = t % 5
        if kind == 0:
            sel = pool if t % 10 == 0 else list(rng.permutation(pool))
        elif kind == 1:
            sel = [int(rng.choice(pool))]
        else:
            sel = [int(s) for s in rng.permutation(pool)[:int(rng.integers(1, len(pool) + 1))]]
        K = int(rng.choice([1, 2, 5, 7]))
        valid = None
        if rng.random() < 0.2:
            valid = rng.integers(0, K + 1, size=len(sel))
        call(events, sel, K, valid)
    cut = set(int(s) for s in np.flatnonzero(book.fresh))
    if lat:                                        # flush every stream
        call([('end', None)], list(range(n)), lat)
    return calls, [[tuple(q) for q in sq] for sq in seqs], cut


@pytest.fixture(scope='module')
def plans():
    return {}


def get_plan(plans, name):
    if name not in plans:
        case = CASES[name]
        calls, seqs, cut = plan(case)
        frames = max(sum(L for _, L in sq) for sq in seqs) + 1
        supply = synth.synth_input(case.n, frames, case.J, 2, seed=200 + case.seed)     # (n, frames, J, 2)
        plans[name] = (calls, seqs, supply, cut)
    return plans[name]


def drive(case, model, calls, supply):
    """run the schedule on a PoseStream; NaN in every held row -> [(y (m, K, J, 3) numpy, index)], the stream"""
    ps = PoseStream(model, case.n, augment=case.augment, **DS.lists(case.J))
    ps.step = case.start
    dev = torch.device('cuda')
    out = []
    for q, (events, sel, K, valid, src, index, _) in enumerate(calls):
        for kind, ss in events:
            getattr(ps, kind)(ss)
        hold = copy.deepcopy(ps.book).advance_many(K, valid, streams=sel)[1]
        fr = np.full((sel.size, K, case.J, 2), np.nan, dtype=np.float32)
        for i, s in enumerate(sel):
            live = np.flatnonzero(~hold[i])
            fr[i, live] = supply[s, src[i]:src[i] + live.size]
        fr = torch.from_numpy(fr).to(dev)
        everyone = sel.size == case.n and np.array_equal(sel, np.arange(case.n))
        if K == 1 and valid is None and q % 2:
            y, idx = ps.push(fr[:, 0], streams=None if everyone else sel)
            y, idx = y[:, None], idx[:, None]
        else:
            y, idx = ps.push_frames(fr, valid=valid, streams=None if everyone else list(sel))
        assert np.array_equal(idx.numpy(), index), q
        out.append((y.cpu().numpy(), idx.numpy()))
    return out, ps


def sampled(case):
    """the streams compared with fp64: every one up to 16, else the special ones and 12 spread over the rest"""
    if case.n <= 16:
        return tuple(range(case.n))
    return tuple(sorted({SLEEPER, WRAPPER, SHORT} | {int(s) for s in np.linspace(3, case.n - 1, 12)}))


_REF = {}


def reference(name, seqs, supply):
    """fp64 poses of every sequence of the sampled streams: {(s, k): (L, J, 3)}"""
    if name not in _REF:
        case = CASES[name]
        keys = [(s, k) for s in sampled(case) for k, (a, L) in enumerate(seqs[s]) if L > 0]
        got = D.sequence_poses([supply[s, seqs[s][k][0]:seqs[s][k][0] + seqs[s][k][1]] for s, k in keys], case.J,
                               case.fw, case.causal, case.augment, D.symmetry(case.J), D.module(case).state_dict())
        _REF[name] = dict(zip(keys, got))
    return _REF[name]


def compare(name, calls, seqs, supply, cut, out):
    """-> (max error / max |y64|, relative L2, poses): every returned pose of the sampled streams against fp64; each
    sequence's poses come once each, in order, and the flush completes the last one"""
    case = CASES[name]
    ref = reference(name, seqs, supply)
    pick = set(sampled(case))
    got, want = [], []
    seen = {}
    for (events, sel, K, valid, src, index, seq), (y, idx) in zip(calls, out):
        for i, s in enumerate(sel):
            if s not in pick:
                continue
            for k in np.flatnonzero(idx[i] >= 0):
                j = int(idx[i, k])
                key = (int(s), int(seq[i]))
                assert seen.get(key, -1) == j - 1, (key, j)
                seen[key] = j
                got.append(y[i, k])
                want.append(ref[key][j])
    lat = D.latency(case.fw, case.causal)
    for s in pick - cut:
        if seqs[s] and seqs[s][-1][1] and lat:
            assert seen[(s, len(seqs[s]) - 1)] == seqs[s][-1][1] - 1, s
    got, want = np.stack(got), np.stack(want)
    assert np.isfinite(got).all()
    mx, l2 = S.errors(got, want)
    return mx, l2, len(got)


def test_schedule_reaches(plans):
    """ticks of one stream and of every stream, an idle stretch longer than R_max while the others wrap their rings
    at least twice, an end on the stream's own ring wrap, a sequence shorter than the latency, counts from 2^40"""
    assert {c.J for c in CASES.values()} == {15, 16, 17, 19}
    assert any(c.start >= X.BIG for c in CASES.values())
    for name, case in CASES.items():
        calls, seqs, _, _ = get_plan(plans, name)
        R, lat = r_max(case.fw), D.latency(case.fw, case.causal)
        assert any(sel.size == 1 for _, sel, *_ in calls) and any(sel.size == case.n for _, sel, *_ in calls)
        count = np.full(case.n, case.start, dtype=np.int64)
        idle, moved, wrap_end, slept = 0, np.zeros(case.n, dtype=np.int64), False, False
        for events, sel, K, *_ in calls:
            if any(kind == 'end' and ss == [WRAPPER] for kind, ss in events):
                wrap_end |= count[WRAPPER] % R == 0
            if SLEEPER in sel:
                slept |= idle > R and moved.max() >= 2 * R          # the others wrapped their rings twice and more
                moved[:] = 0
                idle = 0
            else:
                idle += 1
            count[sel] += K
            moved[sel] += K
        assert slept and wrap_end, (name, slept, wrap_end)
        if lat > 2:
            assert any(L == 2 for _, L in seqs[SHORT]), name


@pytest.mark.parametrize('name', sorted(CASES))
def test_random_subsets_vs_fp64(name, core, plans):
    case = CASES[name]
    calls, seqs, supply, cut = get_plan(plans, name)
    out, ps = drive(case, D.module(case).cuda(), calls, supply)
    assert np.array_equal(ps.counts, case.start + np.array(
        [sum(K for _, sel, K, *_ in calls if s in sel) for s in range(case.n)]))
    mx, l2, rows = compare(name, calls, seqs, supply, cut, out)
    DS.report('subset %s core %d: max %.2e l2 %.2e | %d poses, %d calls' % (name, core, mx, l2, rows, len(calls)))
    assert mx <= MAX_BAR and l2 <= L2_BAR, (mx, l2)


def test_tf32_random_subsets_vs_fp64(plans):
    name = 'j17_333_c128_n37_aug'
    case = CASES[name]
    calls, seqs, supply, cut = get_plan(plans, name)
    m = engine.set_precision(D.module(case).cuda(), 'tf32')
    out, _ = drive(case, m, calls, supply)
    mx, _, _ = compare(name, calls, seqs, supply, cut, out)
    DS.report('subset tf32 %s: max %.2e' % (name, mx))
    engine.set_precision(m, 'fp32')
    assert mx < TF32_BAR, mx


# ---- the C ABI: bitwise checks ------------------------------------------------------------------------------------
def abi(model):
    dev = torch.device('cuda', 0)
    h = engine.model_handle(model, dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    h.refresh(model, st)
    return h, h.lib, st, dev


def vp(t):
    return C.c_void_p(None if t is None else t.data_ptr())


def host(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    return a, C.c_void_p(a.ctypes.data)


def push_subset(lib, h, state, n, streams, steps, K, x, y, ws, st, fresh=None, hold=None):
    s, sp = host(streams, np.int32)
    t, tp = host(steps, np.int64)
    return lib.gast_stream_push_subset(h.h, vp(state), n, sp, tp, len(s), K, vp(x), vp(y), vp(fresh), vp(hold), vp(ws),
                                       ws.numel() if ws is not None else 0, C.c_void_p(st))


def peek_subset(lib, h, state, n, streams, steps, K, y, ws, st, nbytes=None):
    s, sp = host(streams, np.int32)
    t, tp = host(steps, np.int64)
    return lib.gast_stream_peek_subset(h.h, vp(state), n, sp, tp, len(s), K, vp(y), vp(ws),
                                       ws.numel() if nbytes is None else nbytes, C.c_void_p(st))


def state_rows(case, state, n):
    """{stream: [its input-history row, its row of every slot of every ring]} as float views of `state` (the layout
    of stream_plan in csrc/stream.cuh: 64-float aligned parts after a 256-byte aligned base)"""
    f = state.view(torch.float32) if state.data_ptr() % 256 == 0 else None
    assert f is not None
    k0, J = case.fw[0], case.J
    off = 0

    def take(nf):
        nonlocal off
        o = off
        off += (nf + 63) & ~63
        return o
    xo = take(n * k0 * J * 2)
    rings = []
    for w, d, R, Cw in X.stages(S.Case(J, case.fw, case.ch, n, 1, 0, (), 0)):
        rings.append((take(R * n * J * Cw), R, J * Cw))
    out = {}
    for s in range(n):
        parts = [f[xo + s * k0 * J * 2:xo + (s + 1) * k0 * J * 2]]
        for o, R, row in rings:
            parts += [f[o + (r * n + s) * row:o + (r * n + s + 1) * row] for r in range(R)]
        out[s] = torch.cat(parts).clone()
    return out


def warm_state(case, m, n, steps):
    """a state of n streams after `steps` pushes of a chunk (fresh at step 0) -> (h, lib, st, dev, state)"""
    h, lib, st, dev = abi(m)
    nb = int(lib.gast_stream_state_bytes(h.h, n))
    state = torch.zeros(nb, dtype=torch.uint8, device=dev)
    cb = int(lib.gast_stream_chunk_workspace_bytes(h.h, n, steps))
    ws = torch.empty(cb, dtype=torch.uint8, device=dev)
    x = torch.from_numpy(synth.synth_input(n, steps, case.J, 2, seed=5)).cuda()
    y = torch.empty((n, steps, case.J, 3), device=dev)
    fresh = torch.ones(n, dtype=torch.int32, device=dev)
    assert lib.gast_stream_push_chunk(h.h, vp(state), C.c_int64(0), vp(x), vp(y), n, steps, vp(fresh), vp(None), vp(ws),
                                      cb, C.c_void_p(st)) == 0
    return h, lib, st, dev, state


@pytest.mark.parametrize('order', ['in_order', 'reversed'])
def test_all_streams_at_one_step_bitwise_like_chunk(order, core):
    """listing every stream at one step is the chunk path: the same poses and the same state, bit for bit (in order the
    same kernels without a table; reversed through the table)"""
    case = Case(17, (3, 3, 3), 64, 6, 1, 0, (), 81, False, True)
    m = D.module(case).cuda()
    n, K, J = 2 * case.n, 5, case.J
    h, lib, st, dev, state = warm_state(case, m, n, 30)
    other = state.clone()
    x = torch.from_numpy(synth.synth_input(n, K, J, 2, seed=6)).cuda()
    hold = torch.zeros((n, K), dtype=torch.int32, device=dev)
    hold[1, 2:] = 1
    cb = int(lib.gast_stream_chunk_workspace_bytes(h.h, n, K))
    ws = torch.empty(cb, dtype=torch.uint8, device=dev)
    y = torch.empty((n, K, J, 3), device=dev)
    assert lib.gast_stream_push_chunk(h.h, vp(state), C.c_int64(30), vp(x), vp(y), n, K, vp(None), vp(hold), vp(ws), cb,
                                      C.c_void_p(st)) == 0
    perm = np.arange(n) if order == 'in_order' else np.arange(n)[::-1].copy()
    sb = int(lib.gast_stream_subset_workspace_bytes(h.h, n, K))
    ws2 = torch.empty(sb, dtype=torch.uint8, device=dev)
    y2 = torch.empty((n, K, J, 3), device=dev)
    pt = torch.from_numpy(perm).to(dev)
    assert push_subset(lib, h, other, n, perm, np.full(n, 30), K, x[pt].contiguous(), y2, ws2, st,
                       hold=hold[pt].contiguous()) == 0
    assert torch.equal(y2, y[pt])
    assert torch.equal(other, state)


def test_peek_subset_bitwise_like_peek(core):
    """on a lockstep state: every stream in order, reversed, and a partial subset against gast_stream_peek"""
    case = Case(17, (3, 3, 3, 3), 32, 5, 1, 0, (), 83, False, False)
    m = D.module(case).cuda()
    n, J, lat = case.n, case.J, D.latency(case.fw, False)
    h, lib, st, dev, state = warm_state(case, m, n, 50)
    before = state.clone()
    for K in (1, lat):
        cb = int(lib.gast_stream_chunk_workspace_bytes(h.h, n, K))
        ws = torch.empty(cb, dtype=torch.uint8, device=dev)
        y = torch.empty((n, K, J, 3), device=dev)
        assert lib.gast_stream_peek(h.h, vp(state), C.c_int64(50), vp(y), n, K, vp(ws), cb, C.c_void_p(st)) == 0
        for sel in (np.arange(n), np.arange(n)[::-1].copy(), np.array([3, 0])):
            ws2 = torch.empty(int(lib.gast_stream_subset_workspace_bytes(h.h, sel.size, K)), dtype=torch.uint8,
                              device=dev)
            y2 = torch.empty((sel.size, K, J, 3), device=dev)
            assert peek_subset(lib, h, state, n, sel, np.full(sel.size, 50), K, y2, ws2, st) == 0
            assert torch.equal(y2, y[torch.from_numpy(sel).to(dev)]), (K, sel)
            assert torch.equal(state, before)


def test_unlisted_streams_and_peeked_state_unchanged(core):
    """a subset push changes no byte of an unlisted stream; a subset peek changes no byte of the state"""
    case = Case(16, (3, 5, 3), 32, 7, 1, 0, (), 85, False, False)
    m = D.module(case).cuda()
    n, J = case.n, case.J
    h, lib, st, dev, state = warm_state(case, m, n, 12)
    steps = np.array([12, 12, 12])
    sel = np.array([5, 1, 3])
    sb = int(lib.gast_stream_subset_workspace_bytes(h.h, 3, 40))
    ws = torch.empty(sb, dtype=torch.uint8, device=dev)
    for K in (1, 40):                        # 40 frames: more than a ring of 15 slots, every slot rewritten
        before = state_rows(case, state, n)
        x = torch.from_numpy(synth.synth_input(3, K, J, 2, seed=K)).cuda()
        y = torch.empty((3, K, J, 3), device=dev)
        assert push_subset(lib, h, state, n, sel, steps, K, x, y, ws, st) == 0
        after = state_rows(case, state, n)
        for s in range(n):
            assert torch.equal(before[s], after[s]) == (s not in sel), (K, s)
        steps = steps + K
    full = state.clone()
    y = torch.empty((2, 4, J, 3), device=dev)
    assert peek_subset(lib, h, state, n, [1, 6], [steps[1], 12], 4, y, ws, st) == 0
    assert torch.equal(state, full)


# ---- PoseStream ---------------------------------------------------------------------------------------------------
def test_no_streams_bitwise_like_a_stream_without_subsets(core):
    """calls with streams=None on equal counts are the lockstep calls: bit for bit, same step, same launches"""
    case = Case(17, (3, 3, 3), 64, 5, 30, 0, ((7, 'end', (2,)), (12, 'reset', (2,))), 87, False, True)
    m = D.module(case).cuda()
    x = torch.from_numpy(D.frames(case)).cuda()
    a, b = PoseStream(m, case.n, augment=True), PoseStream(m, case.n, augment=True)
    t = 0
    while t < case.T:
        K = 1 + t % 4
        for s in (a, b):
            for tt, kind, ss in case.events:
                if t <= tt < t + K:
                    getattr(s, kind)(list(ss))
        fr = x[t:t + K].transpose(0, 1)
        if K == 1:
            ya, ia = a.push(fr[:, 0])
            yb, ib = b.push(fr[:, 0], streams=None)
        else:
            ya, ia = a.push_frames(fr)
            yb, ib = b.push_frames(fr, streams=None)
        assert torch.equal(ya, yb) and torch.equal(ia, ib) and a.last_launches == b.last_launches, t
        t += K
    assert a.step == b.step == case.T and (b.counts == case.T).all()
    ya, ia = a.peek(5)
    yb, ib = b.peek(5, streams=None)
    sel = torch.from_numpy(ia.numpy() >= 0).cuda()
    assert torch.equal(ia, ib) and torch.equal(ya[sel], yb[sel])


def clone(ps):
    c = copy.copy(ps)
    c.book = copy.deepcopy(ps.book)
    c._state = ps._state.clone()
    c._ws = None
    return c


def test_peek_after_phases_diverged(core):
    """peeks of subsets at unequal counts: the index of the book, and bit for bit a held push_frames of a clone"""
    case = Case(19, (3, 3, 3), 32, 6, 1, 0, (), 89, False, True)
    m = D.module(case).cuda()
    ps = PoseStream(m, case.n, augment=True)
    rng = np.random.default_rng(3)
    supply = torch.from_numpy(synth.synth_input(case.n, 400, case.J, 2, seed=9)).cuda()
    lat = ps.latency
    for it in range(30):
        sel = [int(s) for s in rng.permutation(case.n)[:int(rng.integers(1, case.n + 1))]]
        K = int(rng.choice([1, 3, 8]))
        if it == 10:
            ps.end([4])
        if it == 14:
            ps.reset([4])
        ps.push_frames(supply[sel, it * 8:it * 8 + K].contiguous(), streams=sel)
        if it % 3 == 2:
            q = [int(s) for s in rng.permutation(case.n)[:3]]
            for K in (1, lat):
                want = copy.deepcopy(ps.book).peek(K, streams=q)
                before, counts = ps._state.clone(), ps.counts.copy()
                y, idx = ps.peek(K, streams=q)
                assert np.array_equal(idx.numpy(), want), it
                assert torch.equal(ps._state, before) and np.array_equal(ps.counts, counts)
                c = clone(ps)
                yc, ic = c.push_frames(torch.full((3, K, case.J, 2), float('nan'), device='cuda'),
                                       valid=np.zeros(3, dtype=np.int64), streams=q)
                sel_ = torch.from_numpy(idx.numpy() >= 0).cuda()
                assert torch.equal(ic, idx) and torch.equal(yc[sel_], y[sel_]), (it, K)
    assert len(set(ps.counts.tolist())) > 1


def test_two_persons_with_different_valid_frames(core):
    """num_person = 2 of the reference (gen_skes.py:115-130, tools/inference.py:44-56): each person's poses are those of
    that person's valid frames alone, with augmentation; each stream pushes on the frames its person is valid in"""
    case = Case(17, (3, 3, 3), 128, 2, 90, 0, (), 91, False, True)
    m = D.module(case, dilated=True).cuda()
    kpts = D.frames(case)                                     # (T, 2, J, 2)
    valid = [np.ones(case.T, dtype=bool), np.ones(case.T, dtype=bool)]
    valid[1][20:36] = False                                   # the detector lost person 2 twice
    valid[1][60:71] = False
    valid[0][:3] = False
    ps = PoseStream(m, 2, augment=True)
    x = torch.from_numpy(kpts).cuda()
    got = [[], []]
    for t in range(case.T):
        sel = [p for p in (0, 1) if valid[p][t]]
        y, idx = ps.push(x[t, sel], streams=sel)
        for i, p in enumerate(sel):
            if idx[i] >= 0:
                assert idx[i] == len(got[p])
                got[p].append(y[i])
    ps.end()
    y, idx = ps.push_frames(torch.full((2, ps.latency, 17, 2), float('nan'), device='cuda'))
    for p in (0, 1):
        got[p] += [y[p, k] for k in range(ps.latency) if idx[p, k] >= 0]
    kl, kr, jl, jr = D.symmetry(17)
    for p in (0, 1):
        seq = kpts[valid[p], p]
        want = tta.evaluate_sequence(m, seq, kl, kr, jl, jr, causal=False).cpu().numpy()
        g = torch.stack(got[p]).cpu().numpy()
        assert g.shape == want.shape, (p, g.shape)
        w = float(np.abs(g - want).max() / np.abs(want).max())
        DS.report('subset two persons core %d person %d: %.2e' % (core, p, w))
        assert w <= DS.WHOLE_BAR, w


def test_causal_stream_passes_streams():
    case = Case(17, (3, 3, 3), 32, 3, 12, 0, (), 93, True, False)
    m = D.module(case).cuda()
    x = torch.from_numpy(D.frames(case)).cuda()
    a, b = CausalStream(m, 3), CausalStream(m, 1)
    for t in range(case.T):
        ya = a.push(x[t, [2]], streams=[2]) if t % 2 else a.push_frames(x[t:t + 1, [2]].transpose(0, 1), streams=[2])[:, 0]
        yb = b.push(x[t, [2]])
        mx, l2 = S.errors(ya.cpu().numpy(), yb.cpu().double().numpy())
        assert ya.shape == (1, 17, 3) and mx <= MAX_BAR and l2 <= L2_BAR, (t, mx)
    assert a.counts.tolist() == [0, 0, case.T] and a.step == 0


# ---- refusals and launch counts -----------------------------------------------------------------------------------
def test_refusals():
    case = Case(17, (3, 3, 3), 32, 4, 1, 0, (), 95, False, False)
    m = D.module(case).cuda()
    h, lib, st, dev, state = warm_state(case, m, 4, 6)
    n, K, J = 4, 3, 17
    sb = int(lib.gast_stream_subset_workspace_bytes(h.h, 2, K))
    assert sb > 0 and lib.gast_stream_subset_workspace_bytes(h.h, 0, K) == 0
    assert lib.gast_stream_subset_workspace_bytes(h.h, 2, 0) == 0
    assert int(lib.gast_stream_subset_workspace_bytes(h.h, 3, K)) > sb
    ws = torch.empty(sb, dtype=torch.uint8, device=dev)
    x = torch.zeros((2, K, J, 2), device=dev)
    y = torch.empty((2, K, J, 3), device=dev)
    before = state.clone()
    bad = [([0, 0], [6, 6], 'twice'), ([0, 4], [6, 6], 'outside'), ([-1, 1], [6, 6], 'outside'),
           ([0, 1], [6, -1], 'at least 0')]
    for streams, steps, msg in bad:
        assert push_subset(lib, h, state, n, streams, steps, K, x, y, ws, st) != 0
        assert msg in engine.L.last_error(), (streams, engine.L.last_error())
    for mm in (0, 5):
        s, sp = host(list(range(mm)), np.int32)
        t, tp = host([6] * mm, np.int64)
        assert lib.gast_stream_push_subset(h.h, vp(state), n, sp, tp, mm, K, vp(x), vp(y), vp(None), vp(None), vp(ws),
                                           sb, C.c_void_p(st)) != 0
        assert 'm must be in [1, n_streams = 4]' in engine.L.last_error()
    assert torch.equal(state, before)
    assert push_subset(lib, h, before.clone(), n, [3, 1], [6, 6], K, x, y, ws, st) == 0
    small = torch.empty(sb - 1, dtype=torch.uint8, device=dev)
    state2 = before.clone()
    assert push_subset(lib, h, state2, n, [0, 1], [6, 6], K, x, y, small, st) != 0
    assert 'workspace too small' in engine.L.last_error()
    assert torch.equal(state2, before)
    # peek: step >= 1, K in [1, latency], a non-causal model
    yp = torch.empty((2, 13, J, 3), device=dev)
    pw = torch.empty(int(lib.gast_stream_subset_workspace_bytes(h.h, 2, 13)), dtype=torch.uint8, device=dev)
    assert peek_subset(lib, h, before, n, [0, 1], [0, 6], 1, yp, pw, st) != 0 and 'at least 1' in engine.L.last_error()
    assert peek_subset(lib, h, before, n, [0, 1], [6, 6], 14, yp, pw, st) != 0
    assert 'K must be in [1, latency = 13]' in engine.L.last_error()
    assert peek_subset(lib, h, before, n, [1, 1], [6, 6], 1, yp, pw, st) != 0 and 'twice' in engine.L.last_error()
    assert peek_subset(lib, h, before, n, [0, 1], [6, 6], 13, yp, pw, st) == 0
    hc = abi(D.module(case._replace(causal=True)).cuda())[0]
    assert peek_subset(lib, hc, before, n, [0, 1], [6, 6], 1, yp, pw, st) != 0
    assert 'non-causal' in engine.L.last_error()
    torch.cuda.synchronize()
    # Python
    ps = PoseStream(m, 4)
    for streams in ([], [0, 0], [4], [-1], [0.5]):
        with pytest.raises(engine.GastError, match='streams'):
            ps.push(torch.zeros(max(1, len(streams)), J, 2), streams=streams)
        with pytest.raises(engine.GastError, match='streams'):
            ps.peek(1, streams=streams)
    for frame, streams in ((torch.zeros(3, J, 2), [0, 1]), (torch.zeros(2, 16, 2), [0, 1])):
        with pytest.raises(AssertionError):
            ps.push(frame, streams=streams)
    with pytest.raises(AssertionError):
        ps.push_frames(torch.zeros(2, 4, J, 2), streams=[1])
    with pytest.raises(ValueError):
        ps.push_frames(torch.zeros(2, 4, J, 2), valid=[1, 2, 3], streams=[0, 1])
    ps.push(torch.zeros(2, J, 2), streams=[0, 1])
    cs = PoseStream(D.module(case._replace(causal=True)).cuda(), 2)
    with pytest.raises(engine.GastError, match='non-causal'):
        cs.peek(1, streams=[0])


def test_launches_do_not_depend_on_n_m_k():
    case = Case(17, (3, 3, 3), 128, 1, 1, 0, (), 9, False, False)
    m = D.module(case).cuda()
    counts = {}
    for n in (4, 64):
        for aug in (False, True):
            ps = PoseStream(m, n, augment=aug)
            ps.push_frames(torch.zeros(n, 20, 17, 2, device='cuda'))
            counts['chunk', n, aug] = ps.last_launches
            for mm in (1, 3):
                for K in (1, 5):
                    ps.push_frames(torch.zeros(mm, K, 17, 2, device='cuda'), streams=list(range(n - mm, n)))
                    counts['push', n, mm, K, aug] = ps.last_launches
                    ps.peek(K, streams=list(range(mm)))
                    counts['peek', n, mm, K, aug] = ps.last_launches
    for aug in (False, True):
        for what in ('push', 'peek'):
            assert len({c for k, c in counts.items() if k[0] == what and k[-1] == aug}) == 1, counts
        assert counts['push', 4, 1, 1, aug] == counts['chunk', 4, aug], counts
    assert counts['push', 4, 1, 1, True] == counts['push', 4, 1, 1, False] + 2, counts
