"""GPU: K frames per stream in one call (gast_b200.realtime.PoseStream.push_frames, C ABI gast_stream_push_chunk) and
bounded-memory whole-sequence lifting (gast_b200.realtime.lift_sequences), on both GEMM cores:
  * the delayed-stream matrix of tests/test_gpu_zz_delayed_stream.py pushed in chunks of 1, 2, 7, 64, R - 1 and R + 1
    frames (R = the largest ring; also 300 for the 243-frame model) interleaved with single pushes, chunks cut at
    every reset, ends inside chunks given as `valid`, NaN in the rows of held frames; against the fp64 reference;
  * lift_sequences against the unmodified reference's goldens and against tta.evaluate_sequence;
  * the C ABI at K = 1 against gast_stream_push_ex, bitwise equality of the dilated and Optimized1f handles, the
    refusals, and launch counts that depend on neither n nor K.
The bars are those of the delayed-stream file.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from gast_b200 import engine, tta
from gast_b200.realtime import CausalStream, PoseStream, lift_sequences
import delayedref as D
import streamref as S
import test_gpu_zz_delayed_stream as DS

pytestmark = pytest.mark.gpu

Case = D.Case


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def largest_ring(fw):
    return S.receptive_field(fw[:-1]) * fw[-1]


def chunk_lengths(case):
    """longest first, so that a reset-free stretch starts with the longest chunk that fits"""
    R = largest_ring(case.fw)
    out = [300] if S.receptive_field(case.fw) == 243 else []
    return out + [R + 1, R - 1, 64, 7, 2, 1]


def chunk_plan(case):
    """[(t0, K, single)]: every third call a single `push`, the others chunks cycling through chunk_lengths from its
    start at every reset; a chunk takes the next length of the cycle that fits before the next reset (or T)"""
    cuts = sorted({t for t, kind, _ in case.events if kind == 'reset' and t > 0} | {case.T})
    lengths = chunk_lengths(case)
    out, t0, call, c = [], 0, 0, 0
    while t0 < case.T:
        if t0 in cuts:
            c = 0
        room = min(t for t in cuts if t > t0) - t0
        if call % 3 == 2:
            K, single = 1, True
        else:
            fits = [j for j in range(len(lengths)) if lengths[(c + j) % len(lengths)] <= room]
            K = lengths[(c + fits[0]) % len(lengths)] if fits else room
            c += (fits[0] + 1) if fits else 0
            single = False
        call += 1
        out.append((t0, K, single))
        t0 += K
    return out


def push_chunks(case, model, x=None):
    """push every frame of `case` by chunk_plan; ends inside a chunk become `valid`, ends at a chunk start without a
    reset there become valid = 0; NaN in the rows of held frames -> (poses (n, T, J, 3) numpy, index (n, T), the
    stream, chunk sizes used)"""
    x = torch.from_numpy(D.frames(case) if x is None else x).cuda()
    ps = PoseStream(model, case.n, augment=case.augment, **DS.lists(case.J))
    ps.step = case.start
    ys, idx, used = [], [], []
    for t0, K, single in chunk_plan(case):
        here = [(kind, ss) for tt, kind, ss in case.events if tt == t0]
        valid = np.full(case.n, K, dtype=np.int64)
        if single or any(kind == 'reset' for kind, _ in here):
            for kind, ss in here:
                getattr(ps, kind)(None if ss is None else list(ss))
        else:
            for _, ss in here:
                valid[list(range(case.n)) if ss is None else list(ss)] = 0
        for tt, kind, ss in case.events:
            if t0 < tt < t0 + K:
                assert kind == 'end'
                sel = list(range(case.n)) if ss is None else list(ss)
                valid[sel] = np.minimum(valid[sel], tt - t0)
        if single:
            held = torch.from_numpy((ps.book.left >= 0) & ~ps.book.fresh).cuda()
            frame = torch.where(held[:, None, None], torch.full_like(x[t0], float('nan')), x[t0])
            y, i = ps.push(frame)
            y, i = y[:, None], i[:, None]
        else:
            hold = copy.deepcopy(ps.book).advance_many(K, valid)[1]
            fr = x[t0:t0 + K].transpose(0, 1)
            fr = torch.where(torch.from_numpy(hold).cuda()[:, :, None, None], torch.full_like(fr, float('nan')), fr)
            y, i = ps.push_frames(fr, valid=None if (valid == K).all() else valid)
        assert y.shape == (case.n, K, case.J, 3) and i.shape == (case.n, K)
        ys.append(y)
        idx.append(i)
        used.append(K)
    assert ps.step == case.start + case.T
    return torch.cat(ys, 1).cpu().numpy(), torch.cat(idx, 1).numpy(), ps, used


def without_resets(case):
    """the case with its ends only, long enough for chunks of R + 1 and R - 1 in one stretch"""
    R = largest_ring(case.fw)
    return case._replace(events=tuple(e for e in case.events if e[1] == 'end'), T=max(case.T, 2 * R + 10))


# the resets of the matrix leave no stretch of R + 1 frames in most cases: the same geometries without them
LONG = {name + '_ends_only': without_resets(DS.CASES[name])
        for name in ('j17_333_c128_n37_aug', 'j16_353_c32_n16', 'j19_3333_c16_n7_aug')}
ALL = dict(DS.CASES, **LONG)


@pytest.mark.parametrize('name', sorted(ALL))
def test_chunks_vs_fp64(name, core):
    case = ALL[name]
    got, idx, _, used = push_chunks(case, D.module(case).cuda())
    for s in range(case.n):
        assert np.array_equal(idx[s], D.expected_index(case, s)), s
    picked = DS.sample(case)
    ref, ridx = D.reference(case, picked)
    assert np.array_equal(idx[list(picked)], ridx)
    assert np.isfinite(got[list(picked)][ridx >= 0]).all()
    mx, l2 = D.errors(got[list(picked)], ref, ridx)
    DS.report('chunks %s core %d: max %.2e l2 %.2e | %d of %d streams, chunks %s'
              % (name, core, mx, l2, len(picked), case.n, sorted(set(used))))
    assert mx <= DS.MAX_BAR and l2 <= DS.L2_BAR, (mx, l2)


def test_chunk_matrix_reaches():
    """chunks of R - 1 and R + 1 wherever a reset-free stretch holds them, single pushes and chunks of 1, 2 and 7 in
    every case, one chunk longer than 243 frames for the 243-frame model, ends inside chunks"""
    both = 0
    for name, case in ALL.items():
        plan = chunk_plan(case)
        used = {K for _, K, _ in plan}
        assert {1, 2, 7} <= used and any(s for _, _, s in plan), (name, used)
        R = largest_ring(case.fw)
        both += {R - 1, R + 1} <= used
        if S.receptive_field(case.fw) == 243:
            assert max(used) > 243, used
        inside = [t for t, kind, _ in case.events if kind == 'end' and any(t0 < t < t0 + K for t0, K, _ in plan)]
        assert inside or name == 'j15_53_c48_n9_aug', name
    assert both >= 3, both


@pytest.mark.parametrize('name', golden_names('delayed_'))
def test_lift_sequences_goldens(name, core):
    """the unmodified reference's whole-sequence poses, all sequences on one stream, chunks shorter than the longest"""
    g = load_golden(name)
    meta = g['meta']
    lengths = meta['lengths']
    case = Case(meta['J'], tuple(meta['filter_widths']), meta['channels'], 1, 1, 0, (), meta['seed'], meta['causal'],
                meta['augment'])
    cuts = np.cumsum([0] + lengths)
    seqs = [g['x'][cuts[k]:cuts[k + 1]] for k in range(len(lengths))]
    chunk = max(lengths) // 2 - 1
    out = lift_sequences(D.module(case).cuda(), seqs, n_streams=1, chunk=chunk, augment=meta['augment'])
    err = max(float(np.abs(o.cpu().numpy() - g['y'][cuts[k]:cuts[k + 1]]).max()) for k, o in enumerate(out))
    DS.report('lift golden %s core %d: max abs %.2e' % (name, core, err))
    assert err < DS.GOLDEN_TOL, err


@pytest.mark.parametrize('fw,ch,causal', [((3, 3, 3), 128, False), ((3, 3, 3, 3), 64, False), ((3, 3, 3), 64, True)])
def test_lift_sequences_equals_evaluate_sequence(fw, ch, causal, core):
    """sequences of different lengths, one shorter than the latency, packed onto two streams, with augment"""
    lengths = [70, 5, 0, 33, 90]
    case = Case(17, fw, ch, 1, sum(lengths), 0, (), 41, causal, True)
    m = D.module(case, dilated=True).cuda()
    x = D.frames(case)[:, 0]
    cuts = np.cumsum([0] + lengths)
    seqs = [x[cuts[k]:cuts[k + 1]] for k in range(len(lengths))]
    out = lift_sequences(m, seqs, n_streams=2, chunk=24, augment=True)
    kl, kr, jl, jr = D.symmetry(17)
    worst = 0.0
    for k, sq in enumerate(seqs):
        assert out[k].shape == (lengths[k], 17, 3)
        if not lengths[k]:
            continue
        want = tta.evaluate_sequence(m, sq, kl, kr, jl, jr, causal=causal).cpu().numpy()
        worst = max(worst, float(np.abs(out[k].cpu().numpy() - want).max() / np.abs(want).max()))
    DS.report('lift vs evaluate_sequence %s c%d causal %d core %d: %.2e' % (fw, ch, causal, core, worst))
    assert worst <= DS.WHOLE_BAR, worst


def test_lift_sequences_without_augment_equals_forward():
    """augment=False: the plain model forward on the edge-padded sequence"""
    case = Case(17, (3, 3, 3), 32, 1, 50, 0, (), 43, False, False)
    m = D.module(case, dilated=True).cuda()
    seq = D.frames(case)[:, 0]
    out = lift_sequences(m, [seq], n_streams=4, chunk=16)[0]
    pad = (m.receptive_field() - 1) // 2
    with torch.no_grad():
        want = m(torch.from_numpy(np.pad(seq, ((pad, pad), (0, 0), (0, 0)), 'edge')[None]).cuda())[0]
    w = float((out - want).abs().max() / want.abs().max())
    assert w <= DS.WHOLE_BAR, w


def abi(case, model):
    dev = torch.device('cuda', 0)
    h = engine.model_handle(model, dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    h.refresh(model, st)
    return h, h.lib, st, dev


def test_abi_chunk_of_one_equals_push_ex(core):
    """gast_stream_push_chunk with K = 1 against gast_stream_push_ex, frame by frame, with fresh and hold"""
    case = Case(17, (3, 3, 3), 64, 5, 40, 0, (), 47, False, False)
    m = D.module(case).cuda()
    h, lib, st, dev = abi(case, m)
    n, J = case.n, case.J
    nb = int(lib.gast_stream_state_bytes(h.h, n))
    wb = int(lib.gast_stream_workspace_bytes(h.h, n))
    cb = int(lib.gast_stream_chunk_workspace_bytes(h.h, n, 1))
    assert nb > 0 and wb > 0 and cb > 0
    x = torch.from_numpy(D.frames(case)).cuda()
    fresh = torch.ones(n, dtype=torch.int32, device=dev)
    hold = torch.tensor([0, 0, 1, 1, 0], dtype=torch.int32, device=dev)
    outs = []
    for chunked in (False, True):
        state = torch.empty(nb, dtype=torch.uint8, device=dev)
        ws = torch.empty(cb if chunked else wb, dtype=torch.uint8, device=dev)
        ys = []
        for t in range(case.T):
            y = torch.empty((n, J, 3), device=dev)
            fp = C.c_void_p(fresh.data_ptr() if t == 0 else None)
            hp = C.c_void_p(hold.data_ptr() if t >= 25 else None)
            if chunked:
                rc = lib.gast_stream_push_chunk(h.h, C.c_void_p(state.data_ptr()), C.c_int64(t), C.c_void_p(x[t].data_ptr()),
                                                C.c_void_p(y.data_ptr()), n, 1, fp, hp, C.c_void_p(ws.data_ptr()),
                                                ws.numel(), C.c_void_p(st))
            else:
                rc = lib.gast_stream_push_ex(h.h, C.c_void_p(state.data_ptr()), C.c_int64(t), C.c_void_p(x[t].data_ptr()),
                                             C.c_void_p(y.data_ptr()), n, fp, hp, C.c_void_p(ws.data_ptr()), ws.numel(),
                                             C.c_void_p(st))
            assert rc == 0
            ys.append(y)
        outs.append(torch.stack(ys).cpu().numpy())
    mx, l2 = S.errors(outs[1], outs[0].astype(np.float64))
    DS.report('abi K=1 vs push_ex core %d: max %.2e l2 %.2e' % (core, mx, l2))
    assert mx <= DS.MAX_BAR and l2 <= DS.L2_BAR, (mx, l2)


def test_abi_refusals():
    case = Case(17, (3, 3, 3), 32, 3, 4, 0, (), 49, False, False)
    m = D.module(case).cuda()
    h, lib, st, dev = abi(case, m)
    n, K = case.n, 4
    nb = int(lib.gast_stream_state_bytes(h.h, n))
    cb = int(lib.gast_stream_chunk_workspace_bytes(h.h, n, K))
    assert cb > int(lib.gast_stream_chunk_workspace_bytes(h.h, n, 1)) > 0
    assert lib.gast_stream_chunk_workspace_bytes(h.h, n, 0) == 0
    assert lib.gast_stream_chunk_workspace_bytes(h.h, n, 2 ** 30) == 0          # more than 2^31 positions
    state = torch.empty(nb, dtype=torch.uint8, device=dev)
    ws = torch.empty(cb, dtype=torch.uint8, device=dev)
    x = torch.zeros((n, K, case.J, 2), device=dev)
    y = torch.empty((n, K, case.J, 3), device=dev)
    fresh = torch.ones(n, dtype=torch.int32, device=dev)

    def call(k, nbytes):
        return lib.gast_stream_push_chunk(h.h, C.c_void_p(state.data_ptr()), C.c_int64(0), C.c_void_p(x.data_ptr()),
                                          C.c_void_p(y.data_ptr()), n, k, C.c_void_p(fresh.data_ptr()), C.c_void_p(None),
                                          C.c_void_p(ws.data_ptr()), nbytes, C.c_void_p(st))
    assert call(K, cb - 1) != 0 and 'workspace too small' in engine.L.last_error()
    assert call(0, cb) != 0 and 'K must be at least 1' in engine.L.last_error()
    assert call(K, cb) == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize('augment', [False, True])
def test_dilated_handle_chunks_bitwise_like_optimized1f(augment, core):
    case = DS.CASES['j16_353_c32_n16']._replace(augment=augment)
    a = push_chunks(case, D.module(case).cuda())[0]
    b = push_chunks(case, D.module(case, dilated=True).cuda())[0]
    idx = np.stack([D.expected_index(case, s) for s in range(case.n)])
    assert np.array_equal(a[idx >= 0], b[idx >= 0]), float(np.nanmax(np.abs(a - b)))


def test_causal_stream_push_frames():
    """CausalStream.push_frames returns the poses of its frames, close to single pushes, for one frame too"""
    case = Case(17, (3, 3, 3), 32, 3, 20, 0, (), 51, True, False)
    m = D.module(case).cuda()
    x = torch.from_numpy(D.frames(case)).cuda()
    a, b = CausalStream(m, case.n), CausalStream(m, case.n)
    ya = torch.stack([a.push(x[t]) for t in range(case.T)], 1)
    yb = torch.cat([b.push_frames(x[0:9].transpose(0, 1)), b.push_frames(x[9:10].transpose(0, 1)),
                    b.push_frames(x[10:20].transpose(0, 1))], 1)
    assert yb.shape == ya.shape
    mx, l2 = S.errors(yb.cpu().numpy(), ya.cpu().double().numpy())
    assert mx <= DS.MAX_BAR and l2 <= DS.L2_BAR, (mx, l2)


def test_refusals_match_push():
    from model.gast_net import SpatioTemporalModel
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from gast_b200 import synth
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    dense = SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], channels=16, dense=True).cuda().eval()
    with pytest.raises(engine.GastError, match='dense'):
        PoseStream(dense, 2)
    case = Case(17, (3, 3, 3), 32, 2, 1, 0, (), 53, False, False)
    m = D.module(case).cuda()
    ps = PoseStream(m, 2)
    for bad in (torch.zeros(2, 0, 17, 2), torch.zeros(3, 4, 17, 2), torch.zeros(2, 4, 16, 2), torch.zeros(2, 17, 2)):
        with pytest.raises(AssertionError):
            ps.push_frames(bad)
    with pytest.raises(AssertionError):
        ps.push(torch.zeros(3, 17, 2))
    with pytest.raises(ValueError):
        ps.push_frames(torch.zeros(2, 4, 17, 2), valid=[1, 5])
    m.train()
    for call in (lambda: ps.push(torch.zeros(2, 17, 2)), lambda: ps.push_frames(torch.zeros(2, 4, 17, 2))):
        with pytest.raises(engine.GastError, match='eval'):
            call()
    m.eval()
    x = torch.from_numpy(D.frames(case._replace(T=12))).cuda()
    ps.push_frames(x[0:3].transpose(0, 1))
    ps.push(x[3])
    DS.X._change('load_state_dict', m, S.Case(17, (3, 3, 3), 32, 2, 30, 0, (), 11))
    for call in (lambda: ps.push(x[4]), lambda: ps.push_frames(x[4:8].transpose(0, 1))):
        with pytest.raises(engine.GastError, match='reset'):
            call()
    ps.reset([0])
    with pytest.raises(engine.GastError, match='reset'):
        ps.push_frames(x[4:8].transpose(0, 1))
    ps.reset()
    y, idx = ps.push_frames(x[4:8].transpose(0, 1))
    assert idx.shape == (2, 4) and ps.last_launches > 0


def test_launches_do_not_depend_on_n_and_k_and_augment_adds_two():
    case = Case(17, (3, 3, 3), 128, 1, 1, 0, (), 9, False, False)
    m = D.module(case).cuda()
    counts = {}
    for n in (1, 64):
        for K in (2, 64):
            for aug in (False, True):
                ps = PoseStream(m, n, augment=aug)
                x = torch.zeros(n, K, 17, 2, device='cuda')
                for _ in range(2):
                    ps.push_frames(x)
                counts[n, K, aug] = ps.last_launches
    for aug in (False, True):
        assert len({c for (n, K, a), c in counts.items() if a == aug}) == 1, counts
    assert counts[1, 2, True] == counts[1, 2, False] + 2, counts
