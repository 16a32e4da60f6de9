"""GPU: the peek of a non-causal stream (gast_b200.realtime.PoseStream.peek, C ABI gast_stream_peek), on both GEMM cores:
  * the non-causal cases of the delayed-stream matrix of tests/test_gpu_zz_delayed_stream.py (J = 15/16/17/19, augment
    on and off, a first width of 5, a 5-tap stage, the 243-frame model over several ring revolutions, 640 streams),
    peeked at every push (at sampled pushes for the 243-frame model and the 640 streams) with K cycling through
    latency, 1, latency/2 and latency - 1: the indices against tests/peekref.py for every stream, the poses against
    its fp64 reference on a sample of streams and peek points, and the state bytes unchanged by every peek;
  * against the unmodified reference's poses of every prefix (the peek_* goldens);
  * bitwise against `push_frames` of K held frames on a cloned stream, at every push, on the dilated and the
    Optimized1f handle; K = latency bitwise against `end()` and one `push_frames` flush, and against a flush by single
    pushes to float rounding; later pushes bitwise those of a run without peeks;
  * step counters from 2^40 + phase through the C ABI, a NaN stream gone idle, TF32, launch counts, refusals.

Measured on an H100 80GB HBM3 (400 W power limit), worst over the cases and both GEMM cores, against fp64: max error
/ max |y64| 2.3e-6 (the 243-frame model; 1.4e-6 at most elsewhere), relative L2 1.6e-6; against the peek goldens 9.1e-6
absolute (the 81-frame golden, max |y| 4.5; its own fp32 rounding is 5.5e-6 absolute, tests/test_peekref_cpu.py), at
most 2.6e-6 for the others; TF32 against fp64 9.8e-4 of max |y|.  The bars are about 4x those; the goldens keep the
delayed goldens' 1.6e-5.  The file runs in about 70 s.
"""
import copy
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from gast_b200 import engine
from gast_b200.realtime import CausalStream, PoseStream
import delayedref as D
import peekref as P
import streamref as S
import test_gpu_zz_delayed_stream as DS
import test_gpu_zz_stream_exact as X

pytestmark = pytest.mark.gpu

MAX_BAR = 9e-6                     # max |y - y64| / max |y64|, either GEMM core
L2_BAR = 6.5e-6                    # relative L2 error
GOLDEN_TOL = DS.GOLDEN_TOL         # absolute, against the peek_* goldens (fp32 reference output)
TF32_BAR = 5e-3                    # max |y - y64| / max |y64| in TF32 (DESIGN.md §4.1)

CASES = {k: c for k, c in DS.CASES.items() if not c.causal}
BIG = ('j17_33333_c16_n3', 'j17_333_c32_n640_aug')   # peeked at sampled pushes


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def lat_of(case):
    return D.latency(case.fw, case.causal)


def k_cycle(case):
    lat = lat_of(case)
    return [lat, 1, max(1, lat // 2), max(1, lat - 1)]


def ring_wraps(case):
    """push indices where the largest ring (and so every ring) is back at slot 0"""
    R = S.receptive_field(case.fw)
    return [t for t in range(1, case.T + 1) if (case.start + t) % R == 0]


def peek_points(case):
    """every push for the small cases; for the large ones the events and their neighbours, the ring wraps, the
    latency and twice it, and the end"""
    if case.T <= 150 and case.n * (2 if case.augment else 1) <= 128:
        return list(range(case.T + 1))
    lat = lat_of(case)
    pts = {1, lat - 1, lat, lat + 1, 2 * lat, case.T}
    for t, _, _ in case.events:
        pts |= {t - 1, t, t + 1}
    for t in ring_wraps(case):
        pts |= {t - 1, t, t + 1}
    return sorted(p for p in pts if 0 <= p <= case.T)


def fp64_points(case):
    """the peek points compared with fp64: events, ring wraps, the latency and the end (at most 16)"""
    lat = lat_of(case)
    pts = {lat - 1, lat + 1, case.T} | {t for t, _, _ in case.events} | {t + 1 for t, k, _ in case.events if k == 'end'}
    pts |= set(ring_wraps(case)[:2])
    return sorted(p for p in pts if 1 <= p <= case.T)


def fp64_streams(case):
    """at most 6 of the delayed-stream file's sampled streams, spread over the sample, with the first and last"""
    picked = DS.sample(case)
    if len(picked) <= 6:
        return picked
    sel = {picked[0], picked[-1]} | {picked[int(i)] for i in np.linspace(0, len(picked) - 1, 6)[1:-1]}
    return tuple(sorted(sel))


@functools.lru_cache(maxsize=None)
def fp64_full(name):
    case = CASES[name]
    return P.peeks(case, D.frames(case), fp64_streams(case), fp64_points(case), lat_of(case))


def fp64(name, K):
    """fp64 peeks of K frames at fp64_points on fp64_streams (shared by both cores): the first K rows of the peek of
    latency frames"""
    y, idx = fp64_full(name)
    return y[:, :, :K], idx[:, :, :K]


def clone(ps):
    """a stream with the same state bytes, book and step (its own state tensor)"""
    c = copy.copy(ps)
    c.book = copy.deepcopy(ps.book)
    c._state = ps._state.clone()
    c._ws = None
    return c


def nan_frames(ps, K):
    return torch.full((ps.n, K, ps.J, ps.F), float('nan'), device='cuda')


def drive(case, model, points, ks, on_peek=None, x=None, stream_cls=PoseStream):
    """push every frame of `case` (NaN in held rows) with its events, peeking K = ks[i % len(ks)] at the i-th peek point
    (after the events of that push, before the push; point T after the last push).  Every peek must leave the state
    bytes and the book unchanged.  on_peek(ps, t, K, y, index) is called after each peek.
    -> (push poses (n, T, J, 3) numpy, peeks {t: (K, y numpy, index)}, the stream)"""
    x = torch.from_numpy(D.frames(case) if x is None else x).cuda()
    ps = stream_cls(model, case.n, augment=case.augment, **DS.lists(case.J))
    ps.step = case.start
    ys, peeks = [], {}
    points = set(points)
    for t in range(case.T + 1):
        for tt, kind, ss in case.events:
            if tt == t:
                getattr(ps, kind)(None if ss is None else list(ss))
        if t in points:
            K = ks[len(peeks) % len(ks)]
            before = None if ps._state is None else ps._state.clone()
            book = (ps.book.fresh.copy(), ps.book.length.copy(), ps.book.left.copy())
            step = ps.step
            y, idx = ps.peek(K)
            assert y.shape == (case.n, K, case.J, 3) and idx.shape == (case.n, K)
            if before is not None:
                assert torch.equal(ps._state, before), t
            assert ps.step == step and all(np.array_equal(a, b) for a, b in
                                           zip(book, (ps.book.fresh, ps.book.length, ps.book.left))), t
            if on_peek is not None:
                on_peek(ps, t, K, y, idx)
            peeks[t] = (K, y.cpu().numpy(), idx.numpy())
        if t == case.T:
            break
        held = torch.from_numpy((ps.book.left >= 0) & ~ps.book.fresh).cuda()
        frame = torch.where(held[:, None, None], torch.full_like(x[t], float('nan')), x[t])
        ys.append(ps.push(frame)[0])
    return torch.stack(ys, 1).cpu().numpy(), peeks, ps


def test_peek_matrix_reaches():
    """J = 15/16/17/19, augment on and off, first width 5, a 5-tap stage, the 243-frame model over three ring
    revolutions, more than 1024 library streams, step counters from 2^40; K from 1 to latency"""
    assert {c.J for c in CASES.values()} == {15, 16, 17, 19}
    assert {c.augment for c in CASES.values()} == {False, True}
    assert any(c.fw[0] == 5 for c in CASES.values()) and any(5 in c.fw[1:] for c in CASES.values())
    assert any(S.receptive_field(c.fw) == 243 and c.T > 3 * 243 for c in CASES.values())
    assert any(c.n * (2 if c.augment else 1) > 1024 for c in CASES.values())
    assert any(c.start >= X.BIG for c in CASES.values())
    for name, c in CASES.items():
        assert {1, lat_of(c)} <= set(k_cycle(c))
        assert (name in BIG) == (peek_points(c) != list(range(c.T + 1))), name
        assert len(fp64_points(c)) <= 16 and len(fp64_streams(c)) <= 6


@pytest.mark.parametrize('name', sorted(CASES))
def test_peek_vs_fp64(name, core):
    case = CASES[name]
    streams, pts = list(fp64_streams(case)), fp64_points(case)
    ks = sorted(set(k_cycle(case)))
    got = {K: np.full(fp64(name, K)[0].shape, np.nan) for K in ks}

    def at_fp64_points(ps, t, K, y, idx):
        """peek every K of the cycle at the fp64 points (a peek changes nothing, so they may follow each other)"""
        if t not in pts:
            return
        q = pts.index(t)
        for KK in ks:
            yy, ii = (y, idx) if KK == K else ps.peek(KK)
            assert np.array_equal(ii.numpy()[streams], fp64(name, KK)[1][:, q]), (t, KK)
            got[KK][:, q] = yy.cpu().numpy()[streams]

    _, peeks, _ = drive(case, D.module(case).cuda(), sorted(set(peek_points(case)) | set(pts)), k_cycle(case),
                        on_peek=at_fp64_points)
    for t, (K, _, idx) in peeks.items():                      # the indices of every stream at every peek
        want = np.stack([P.expected_index(case, s, t, K) for s in range(case.n)])
        assert np.array_equal(idx, want), t
    worst, rows = [0.0, 0.0], 0
    for K in ks:
        ref, ridx = fp64(name, K)
        assert np.isfinite(got[K][ridx >= 0]).all()
        mx, l2 = P.errors(got[K], ref, ridx)
        worst = [max(worst[0], mx), max(worst[1], l2)]
        rows += int((ridx >= 0).sum())
    DS.report('peek %s core %d: max %.2e l2 %.2e | %d peeks, %d rows of %d streams vs fp64'
              % (name, core, worst[0], worst[1], len(peeks), rows, len(streams)))
    assert rows > 0 and worst[0] <= MAX_BAR and worst[1] <= L2_BAR, worst


@pytest.mark.parametrize('name', golden_names('peek_'))
def test_peek_goldens(name, core):
    """the unmodified reference's poses of every prefix: one stream pushes the sequence and peeks K = latency after
    each prefix"""
    g = load_golden(name)
    meta = g['meta']
    T = len(g['x'])
    case = D.Case(meta['J'], tuple(meta['filter_widths']), meta['channels'], 1, T, 0, (), meta['seed'], False,
                  meta['augment'])
    lat = lat_of(case)
    prefixes = [int(p) for p in g['prefixes']]
    _, peeks, _ = drive(case, D.module(case).cuda(), prefixes, [lat], x=g['x'][:, None].copy())
    err = 0.0
    for q, p in enumerate(prefixes):
        _, y, idx = peeks[p]
        sel = idx[0] >= 0
        assert np.array_equal(sel, np.isfinite(g['y'][q, :, 0, 0])), p
        err = max(err, float(np.abs(y[0][sel] - g['y'][q][sel]).max()))
    DS.report('peek golden %s core %d: max abs %.2e' % (name, core, err))
    assert err < GOLDEN_TOL, err


def check_against_clones(ps, t, K, y, idx):
    """the peek equals, bit for bit, push_frames of K held frames (valid = 0) on a clone; for K = latency also end() +
    push_frames on a clone, and (to float rounding) end() + K single pushes"""
    sel = torch.from_numpy(idx.numpy() >= 0)
    if not bool(sel.any()):
        return
    a = clone(ps)
    ya, ia = a.push_frames(nan_frames(ps, K), valid=np.zeros(ps.n, dtype=np.int64))
    assert torch.equal(ia, idx), t
    assert torch.equal(ya[sel.cuda()], y[sel.cuda()]), (t, K)
    if K == ps.latency:
        b = clone(ps)
        b.end()
        yb, ib = b.push_frames(nan_frames(ps, K))
        assert torch.equal(ib, idx) and torch.equal(yb[sel.cuda()], y[sel.cuda()]), t
        c = clone(ps)
        c.end()
        yc = torch.stack([c.push(nan_frames(ps, 1)[:, 0])[0] for _ in range(K)], 1)
        mx, l2 = S.errors(yc[sel.cuda()].cpu().numpy(), y[sel.cuda()].cpu().double().numpy())
        assert mx <= MAX_BAR and l2 <= L2_BAR, (t, mx, l2)


@pytest.mark.parametrize('dilated', [False, True], ids=['optimized1f', 'dilated'])
@pytest.mark.parametrize('name', ['j16_353_c32_n16', 'j17_333_c128_n37_aug'])
def test_peek_bitwise_like_held_chunk(name, dilated, core):
    """at every push: the clones of check_against_clones; and the pushes of the run are bitwise those of a run
    without peeks"""
    case = CASES[name]
    m = D.module(case, dilated=dilated).cuda()
    got, peeks, _ = drive(case, m, range(case.T + 1), k_cycle(case), on_peek=check_against_clones)
    plain = DS.push_all(case, m)[0]
    idx = np.stack([D.expected_index(case, s) for s in range(case.n)])
    assert np.array_equal(got[idx >= 0], plain[idx >= 0])


def test_dilated_handle_peeks_bitwise_like_optimized1f(core):
    case = CASES['j19_3333_c16_n7_aug']
    pts = peek_points(case)
    a = drive(case, D.module(case).cuda(), pts, k_cycle(case))[1]
    b = drive(case, D.module(case, dilated=True).cuda(), pts, k_cycle(case))[1]
    for t in pts:
        sel = a[t][2] >= 0
        assert np.array_equal(a[t][1][sel], b[t][1][sel]), t


def abi(model):
    dev = torch.device('cuda', 0)
    h = engine.model_handle(model, dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    h.refresh(model, st)
    return h, h.lib, st, dev


@pytest.mark.parametrize('fw', [(5, 3), (3, 3, 3, 3)])
def test_abi_peek_at_large_steps(fw, core):
    """step counters from 2^40 + phase (X.phase_start: the rings wrap to slot 0 at pushes 1 and R + 1), so that the
    peeked slots wrap: gast_stream_peek against gast_stream_push_chunk of held frames on a copy of the state, at every
    push, and the state bytes unchanged"""
    case = D.Case(17, fw, 32, 3, S.receptive_field(fw) + 12, X.phase_start(fw), (), 71, False, False)
    m = D.module(case).cuda()
    h, lib, st, dev = abi(m)
    n, J, lat = case.n, case.J, lat_of(case)
    nb = int(lib.gast_stream_state_bytes(h.h, n))
    wb = int(lib.gast_stream_workspace_bytes(h.h, n))
    cb = int(lib.gast_stream_chunk_workspace_bytes(h.h, n, lat))
    state = torch.empty(nb, dtype=torch.uint8, device=dev)
    ws = torch.empty(wb, dtype=torch.uint8, device=dev)
    cws = torch.empty(cb, dtype=torch.uint8, device=dev)
    x = torch.from_numpy(D.frames(case)).cuda()
    fresh = torch.ones(n, dtype=torch.int32, device=dev)
    hold = torch.ones((n, lat), dtype=torch.int32, device=dev)
    xs = torch.zeros((n, lat, J, 2), device=dev)
    for t in range(case.T):
        y = torch.empty((n, J, 3), device=dev)
        assert lib.gast_stream_push_ex(h.h, C.c_void_p(state.data_ptr()), C.c_int64(case.start + t),
                                       C.c_void_p(x[t].data_ptr()), C.c_void_p(y.data_ptr()), n,
                                       C.c_void_p(fresh.data_ptr() if t == 0 else None), C.c_void_p(None),
                                       C.c_void_p(ws.data_ptr()), wb, C.c_void_p(st)) == 0
        K = (lat, 1, 3)[t % 3]
        step = case.start + t + 1
        before = state.clone()
        yp = torch.empty((n, K, J, 3), device=dev)
        assert lib.gast_stream_peek(h.h, C.c_void_p(state.data_ptr()), C.c_int64(step), C.c_void_p(yp.data_ptr()), n,
                                    K, C.c_void_p(cws.data_ptr()), cb, C.c_void_p(st)) == 0
        assert torch.equal(state, before), t
        copy_ = state.clone()
        yc = torch.empty((n, K, J, 3), device=dev)
        assert lib.gast_stream_push_chunk(h.h, C.c_void_p(copy_.data_ptr()), C.c_int64(step), C.c_void_p(xs.data_ptr()),
                                          C.c_void_p(yc.data_ptr()), n, K, C.c_void_p(None),
                                          C.c_void_p(hold.data_ptr()), C.c_void_p(cws.data_ptr()), cb,
                                          C.c_void_p(st)) == 0
        assert torch.equal(yp, yc), (t, K)


def test_nan_stream_gone_idle_leaves_others_alone():
    """a stream that pushed NaN frames, ended and went idle does not change the other streams' peeks"""
    case = D.Case(17, (3, 3, 3), 64, 5, 40, 0, ((6, 'end', (2,)),), 73, False, True)
    m = D.module(case).cuda()
    x = D.frames(case)
    bad = x.copy()
    bad[:6, 2] = np.nan
    pts = list(range(20, case.T + 1))
    a = drive(case, m, pts, k_cycle(case), x=x)[1]
    b = drive(case, m, pts, k_cycle(case), x=bad)[1]
    others = [0, 1, 3, 4]
    for t in pts:
        assert (b[t][2][2] == -1).all()
        assert np.array_equal(a[t][1][others], b[t][1][others]), t
        assert np.isfinite(b[t][1][others][b[t][2][others] >= 0]).all()


def test_tf32_peek_vs_fp64():
    name = 'j17_333_c128_n37_aug'
    case = CASES[name]
    m = engine.set_precision(D.module(case).cuda(), 'tf32')
    streams, pts = list(fp64_streams(case)), fp64_points(case)
    lat = lat_of(case)
    got = np.full(fp64(name, lat)[0].shape, np.nan)

    def keep(ps, t, K, y, idx):
        if t in pts:
            got[:, pts.index(t)] = y.cpu().numpy()[streams]

    drive(case, m, pts, [lat], on_peek=keep)
    ref, ridx = fp64(name, lat)
    mx, _ = P.errors(got, ref, ridx)
    DS.report('peek tf32 %s: max %.2e' % (name, mx))
    assert mx < TF32_BAR, mx
    engine.set_precision(m, 'fp32')


def test_launches_do_not_depend_on_n_and_k_and_augment_adds_two():
    case = D.Case(17, (3, 3, 3), 128, 1, 1, 0, (), 9, False, False)
    m = D.module(case).cuda()
    counts = {}
    for n in (1, 64):
        for K in (1, 7, 13):
            for aug in (False, True):
                ps = PoseStream(m, n, augment=aug)
                ps.push_frames(torch.zeros(n, 20, 17, 2, device="cuda"))
                ps.peek(K)
                counts[n, K, aug] = ps.last_launches
    for aug in (False, True):
        assert len({c for (n, K, a), c in counts.items() if a == aug}) == 1, counts
    assert counts[1, 1, True] == counts[1, 1, False] + 2, counts
    ps = PoseStream(m, 2)
    ps.reset()
    y, idx = ps.peek()                                      # nothing pushed: nothing due, no library call
    assert (idx.numpy() == -1).all() and ps.last_launches == 0


def test_refusals():
    case = D.Case(17, (3, 3, 3), 32, 2, 12, 0, (), 75, False, False)
    m = D.module(case).cuda()
    causal = D.module(case._replace(causal=True)).cuda()
    for s in (PoseStream(causal, 2), CausalStream(causal, 2)):
        with pytest.raises(engine.GastError, match='non-causal'):
            s.peek(1)
    ps = PoseStream(m, 2)
    x = torch.from_numpy(D.frames(case)).cuda()
    ps.push_frames(x[0:5].transpose(0, 1))
    for K in (0, 14, -1):
        with pytest.raises(engine.GastError, match='latency'):
            ps.peek(K)
    m.train()
    with pytest.raises(engine.GastError, match='eval'):
        ps.peek()
    m.eval()
    ps.peek()
    DS.X._change('load_state_dict', m, S.Case(17, (3, 3, 3), 32, 2, 30, 0, (), 11))
    with pytest.raises(engine.GastError, match='reset'):
        ps.peek()
    ps.reset()
    y, idx = ps.peek()
    assert (idx.numpy() == -1).all()
    # the C ABI
    h, lib, st, dev = abi(m)
    n, lat = 2, 13
    cb = int(lib.gast_stream_chunk_workspace_bytes(h.h, n, lat))
    state = torch.zeros(int(lib.gast_stream_state_bytes(h.h, n)), dtype=torch.uint8, device=dev)
    ws = torch.empty(cb, dtype=torch.uint8, device=dev)
    y = torch.empty((n, lat, 17, 3), device=dev)

    def call(hh, step, K, nbytes):
        return lib.gast_stream_peek(hh, C.c_void_p(state.data_ptr()), C.c_int64(step), C.c_void_p(y.data_ptr()), n, K,
                                    C.c_void_p(ws.data_ptr()), nbytes, C.c_void_p(st))
    assert call(h.h, 5, lat, cb) == 0
    assert call(h.h, 5, 0, cb) != 0 and 'K must be in [1, latency = 13]' in engine.L.last_error()
    assert call(h.h, 5, lat + 1, cb) != 0 and 'K must be in' in engine.L.last_error()
    assert call(h.h, 0, lat, cb) != 0 and 'step' in engine.L.last_error()
    assert call(h.h, 5, lat, cb - 1) != 0 and 'workspace too small' in engine.L.last_error()
    assert call(h.h, 5, 1, int(lib.gast_stream_chunk_workspace_bytes(h.h, n, 1))) == 0     # a smaller K needs less
    hc = abi(causal)[0]
    assert call(hc.h, 5, 1, cb) != 0 and 'non-causal' in engine.L.last_error()
    torch.cuda.synchronize()
