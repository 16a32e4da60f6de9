"""GPU: the delayed stream (gast_b200.realtime.PoseStream, C ABI gast_stream_push_ex) of causal and non-causal models,
with and without test-time augmentation, on both GEMM cores:
  * against the unmodified reference's whole-sequence poses (the delayed_* goldens: UnchunkedGenerator + evaluate);
  * against the fp64 reference of tests/delayedref.py over a matrix of ring geometries, joint counts, stream counts
    and step counters, with staggered starts, ends and resets (ends on ring wraps and tile boundaries, end then reset
    on consecutive pushes, resets during a pending tail, sequences shorter than the latency, idle streams);
  * against the GPU whole-sequence forward with TTA (gast_b200.tta.evaluate_sequence).
The rows of held streams are NaN in every push: a held stream must not read them.

Measured on an H100 80GB HBM3 (400 W power limit), worst over the matrix and both GEMM cores, against fp64: max error
/ max |y64| 2.1e-6 (the 243-frame model; 1.4e-6 at most elsewhere), relative L2 1.5e-6; against evaluate_sequence
1.2e-6 (FFMA core); against the goldens 4.1e-6 absolute (their own fp32 rounding is up to 3e-6 of max |y|,
tests/test_delayedref_cpu.py).  The bars are about 4x those.  The file runs in about 70 s.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from gast_b200 import engine, synth, tta
from gast_b200.realtime import CausalStream, PoseStream
import delayedref as D
import streamref as S
import test_gpu_zz_stream_exact as X

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')   # optional directory for the measured errors of these tests

GOLDEN_TOL = 1.6e-5                # absolute, against the delayed_* goldens (fp32 reference output)
MAX_BAR = 9e-6                     # max |y - y64| / max |y64|, either GEMM core
L2_BAR = 6e-6                      # relative L2 error
WHOLE_BAR = 5e-6                   # max |y - y_whole| / max |y_whole|: stream against evaluate_sequence

Case = D.Case
J17_EVENTS = (
    (5, 'end', (3,)), (8, 'reset', (3,)),                   # a 5-frame sequence (< latency 13), reset in its tail
    (12, 'reset', (6, 7)),                                  # staggered starts on both sides of the first frame tile
    (20, 'end', (13, 14)), (21, 'reset', (13,)),            # end then reset on consecutive pushes
    (27, 'end', (0, 36)),                                   # ends where the 27-slot ring wraps to slot 0
    (30, 'end', None), (44, 'reset', None),                 # every stream ends, idles, restarts
    (54, 'end', (20,)), (55, 'reset', (21,)))
CASES = {
    # 6 frame tiles (ragged tail), several flat tiles, mix tail blocks; augment on 74 library streams, and off
    'j17_333_c128_n37_aug': Case(17, (3, 3, 3), 128, 37, 60, 0, J17_EVENTS, 1, False, True),
    'j17_333_c96_n37': Case(17, (3, 3, 3), 96, 37, 60, 0, J17_EVENTS, 1, False, False),
    # first width 5 (latency 7); 48 channels; starts at 2^40 + phase: pushes 1 and 16 land on slot 0 of the 15-slot ring
    'j15_53_c48_n9_aug': Case(15, (5, 3), 48, 9, 40, X.phase_start((5, 3)),
                              ((1, 'end', (3,)), (3, 'reset', (3,)), (7, 'reset', (4, 5)), (16, 'end', (0, 8)),
                               (17, 'reset', (0,)), (25, 'end', None), (33, 'reset', (1, 2))), 2, False, True),
    # a 5-tap stage (latency 22): ends on the 45-slot wrap and at an exact 128-row tile boundary (streams 7 | 8)
    'j16_353_c32_n16': Case(16, (3, 5, 3), 32, 16, 80, 0,
                            ((10, 'reset', None), (30, 'end', (15,)), (31, 'reset', (15,)), (45, 'end', (7, 8)),
                             (50, 'reset', (8,)), (60, 'end', (0,)), (70, 'end', (1, 2))), 3, False, False),
    # 19 joints, 16 channels, latency 40; 2^40 + phase: pushes 1 and 82 land on slot 0 of the 81-slot ring
    'j19_3333_c16_n7_aug': Case(19, (3, 3, 3, 3), 16, 7, 140, X.phase_start((3, 3, 3, 3)),
                                ((1, 'reset', (0, 6)), (20, 'end', (3,)), (40, 'reset', (3,)), (82, 'end', (1, 2)),
                                 (83, 'reset', (1,)), (100, 'end', None)), 4, False, True),
    # the 243-frame model (latency 121) over more than three revolutions of its 243-slot ring
    'j17_33333_c16_n3': Case(17, (3, 3, 3, 3, 3), 16, 3, 800, 0,
                             ((243, 'end', (1,)), (300, 'reset', (1,)), (301, 'reset', (2,)), (600, 'end', (0,))), 5,
                             False, False),
    # many streams: 1280 library streams with augment (rowdot8_kernel's second grid-stride pass), checked on a sample
    'j17_333_c32_n640_aug': Case(17, (3, 3, 3), 32, 640, 40, 0,
                                 ((9, 'end', (0, 639)), (14, 'reset', tuple(range(300, 340))),
                                  (20, 'end', tuple(range(100, 164))), (27, 'reset', None)), 7, False, True),
    # the reference's real-time model kind (causal, latency 0) with augment, as its helpers run it
    'j17_333_c64_causal_n6_aug': Case(17, (3, 3, 3), 64, 6, 40, 0,
                                      ((5, 'end', (1,)), (9, 'reset', (1,)), (20, 'end', None), (27, 'reset', (0, 2, 4))),
                                      8, True, True),
}


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def lists(J):
    """explicit symmetry lists where the reference has no defaults (J = 15, 16)"""
    if J in (17, 19):
        return {}
    kl, kr, jl, jr = D.symmetry(J)
    return dict(kps_left=kl, kps_right=kr, joints_left=jl, joints_right=jr)


def push_all(case, model, x=None, stream_cls=PoseStream):
    """push every frame of `case` (x (T, n, J, 2), default D.frames) with its events and step counter, NaN in the
    rows of held streams -> (poses (n, T, J, 3) numpy, index (n, T)), the stream"""
    x = torch.from_numpy(D.frames(case) if x is None else x).cuda()
    ps = stream_cls(model, case.n, augment=case.augment, **lists(case.J))
    ps.step = case.start
    ys, idx = [], []
    for t in range(case.T):
        for tt, kind, ss in case.events:
            if tt == t:
                getattr(ps, kind)(None if ss is None else list(ss))
        held = torch.from_numpy((ps.book.left >= 0) & ~ps.book.fresh).cuda()
        frame = torch.where(held[:, None, None], torch.full_like(x[t], float('nan')), x[t])
        y, i = ps.push(frame)
        ys.append(y)
        idx.append(i)
    return torch.stack(ys, 1).cpu().numpy(), torch.stack(idx, 1).numpy(), ps


def sample(case):
    """streams compared with fp64: tile / mix / pass boundaries of the n and (with augment) 2n library streams, and
    every stream with an event"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    resets = tuple((t, ss) for t, _, ss in case.events)
    s = set(X.sample(S.Case(case.J, case.fw, case.ch, case.n, case.T, case.start, resets, case.seed), sms))
    if case.augment and case.n > X.FULL_CHECK:
        s |= {c % case.n for c in X.sample(S.Case(case.J, case.fw, case.ch, 2 * case.n, case.T, case.start, (),
                                                  case.seed), sms)}
    return tuple(sorted(s))


def report(line):
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        with open(os.path.join(REPORT_DIR, 'delayed_stream.txt'), 'a') as f:
            f.write(line + '\n')


def test_case_matrix_reaches():
    """joint counts, a first width of 5, a 5-tap stage, the 243-frame model over three ring revolutions, both step
    counters, both augment settings, causal and not, ends on ring wraps and shorter than the latency"""
    assert {c.J for c in CASES.values()} == {15, 16, 17, 19}
    assert any(c.fw[0] == 5 for c in CASES.values()) and any(5 in c.fw[1:] for c in CASES.values())
    assert any(S.receptive_field(c.fw) == 243 and c.T > 3 * 243 for c in CASES.values())
    assert any(c.start >= X.BIG for c in CASES.values()) and any(c.start == 0 for c in CASES.values())
    assert {c.augment for c in CASES.values()} == {False, True} and {c.causal for c in CASES.values()} == {False, True}
    assert any(c.n * (2 if c.augment else 1) > 1024 for c in CASES.values())
    wrap_end = short = 0
    for c in CASES.values():
        rf, lat = S.receptive_field(c.fw), D.latency(c.fw, c.causal)
        wrap_end += any(k == 'end' and (c.start + t) % rf == 0 for t, k, _ in c.events)
        short += any(0 < te - t0 < lat for s in range(c.n) for t0, te, _ in D.sequences(c, s))
    assert wrap_end >= 3 and short >= 2, (wrap_end, short)


@pytest.mark.parametrize('name', golden_names('delayed_'))
def test_delayed_goldens(name, core):
    """the unmodified reference's whole-sequence poses: each sequence on its own stream, ended after its last frame"""
    g = load_golden(name)
    meta = g['meta']
    lengths = meta['lengths']
    n, T = len(lengths), max(lengths) + D.latency(meta['filter_widths'], meta['causal'])
    events = tuple((L, 'end', (k,)) for k, L in enumerate(lengths))
    case = Case(meta['J'], tuple(meta['filter_widths']), meta['channels'], n, T, 0, events, meta['seed'],
                meta['causal'], meta['augment'])
    cuts = np.cumsum([0] + lengths)
    x = np.zeros((T, n, case.J, 2), dtype=np.float32)
    for k, L in enumerate(lengths):
        x[:L, k] = g['x'][cuts[k]:cuts[k + 1]]
    got, idx, _ = push_all(case, D.module(case).cuda(), x=x)
    err = 0.0
    for k, L in enumerate(lengths):
        sel = idx[k] >= 0
        assert np.array_equal(idx[k][sel], np.arange(L)), (k, idx[k])
        err = max(err, float(np.abs(got[k][sel] - g['y'][cuts[k]:cuts[k + 1]]).max()))
    report('golden %s core %d: max abs %.2e' % (name, core, err))
    assert err < GOLDEN_TOL, err


@pytest.mark.parametrize('name', sorted(CASES))
def test_stream_vs_fp64(name, core):
    case = CASES[name]
    got, idx, _ = push_all(case, D.module(case).cuda())
    for s in range(case.n):
        assert np.array_equal(idx[s], D.expected_index(case, s)), s
    picked = sample(case)
    ref, ridx = D.reference(case, picked)
    assert np.array_equal(idx[list(picked)], ridx)
    assert np.isfinite(got[list(picked)][ridx >= 0]).all()
    mx, l2 = D.errors(got[list(picked)], ref, ridx)
    report('%s core %d: max %.2e l2 %.2e | %d of %d streams vs fp64, %d poses'
           % (name, core, mx, l2, len(picked), case.n, int((ridx >= 0).sum())))
    assert mx <= MAX_BAR and l2 <= L2_BAR, (mx, l2)


@pytest.mark.parametrize('fw,ch,causal', [((3, 3, 3), 128, False), ((3, 3, 3, 3), 64, False), ((3, 3, 3), 64, True)])
def test_whole_sequence_equals_evaluate_sequence(fw, ch, causal, core):
    """one sequence pushed and ended, with augment, equals the GPU whole-sequence forward with TTA"""
    T = 70
    lat = D.latency(fw, causal)
    case = Case(17, fw, ch, 1, T + lat, 0, ((T, 'end', None),), 31, causal, True)
    m = D.module(case, dilated=True).cuda()
    x = D.frames(case)
    got, idx, _ = push_all(case, m, x=x)
    sel = idx[0] >= 0
    assert np.array_equal(idx[0][sel], np.arange(T))
    kl, kr, jl, jr = D.symmetry(17)
    want = tta.evaluate_sequence(m, x[:T, 0], kl, kr, jl, jr, causal=causal).cpu().numpy()
    w = float(np.abs(got[0][sel] - want).max() / np.abs(want).max())
    report('whole sequence %s c%d causal %d core %d: %.2e' % (fw, ch, causal, core, w))
    assert w <= WHOLE_BAR, w


def test_pose_stream_equals_causal_stream_bitwise():
    """PoseStream(causal model, augment=False) returns what CausalStream returns, bit for bit"""
    case = X.CASES['j17_333_c128_n37']
    m = S.module(case).cuda()
    x = torch.from_numpy(S.frames(case)).cuda()
    a, b = CausalStream(m, case.n), PoseStream(m, case.n)
    for t in range(case.T):
        for tt, ss in case.resets:
            if tt == t:
                a.reset(None if ss is None else list(ss))
                b.reset(None if ss is None else list(ss))
        ya = a.push(x[t])
        yb, ib = b.push(x[t])
        assert torch.equal(ya, yb), t
        assert ib.tolist() == [t - max(t0 for t0, _ in S.segments(case, s) if t0 <= t) for s in range(case.n)]


@pytest.mark.parametrize('augment', [False, True])
def test_dilated_noncausal_handle_streams_bitwise_like_optimized1f(augment, core):
    case = CASES['j16_353_c32_n16']._replace(augment=augment)
    a = push_all(case, D.module(case).cuda())[0]
    b = push_all(case, D.module(case, dilated=True).cuda())[0]
    idx = np.stack([D.expected_index(case, s) for s in range(case.n)])
    assert np.array_equal(a[idx >= 0], b[idx >= 0]), float(np.nanmax(np.abs(a - b)))


def test_push_equals_push_ex_without_hold():
    """gast_stream_push is gast_stream_push_ex(hold = NULL) for a causal handle; it refuses a non-causal handle,
    which gast_stream_push_ex accepts with the same state and workspace sizes"""
    case = X.CASES['j15_53_c48_n9']
    m = S.module(case).cuda()
    dev = torch.device('cuda', 0)
    h = engine.model_handle(m, dev)
    lib = h.lib
    st = torch.cuda.current_stream(dev).cuda_stream
    h.refresh(m, st)
    n = case.n
    nb, wb = int(lib.gast_stream_state_bytes(h.h, n)), int(lib.gast_stream_workspace_bytes(h.h, n))
    assert nb > 0 and wb > 0 and lib.gast_stream_latency(h.h) == 0
    x = torch.from_numpy(S.frames(case)).cuda()
    fresh = torch.ones(n, dtype=torch.int32, device=dev)
    outs = []
    for ex in (False, True):
        state = torch.empty(nb, dtype=torch.uint8, device=dev)
        ws = torch.empty(wb, dtype=torch.uint8, device=dev)
        ys = []
        for t in range(case.T):
            y = torch.empty((n, case.J, 3), device=dev)
            fp = C.c_void_p(fresh.data_ptr() if t == 0 else None)
            args = [h.h, C.c_void_p(state.data_ptr()), C.c_int64(case.start + t), C.c_void_p(x[t].data_ptr()),
                    C.c_void_p(y.data_ptr()), n, fp]
            if ex:
                rc = lib.gast_stream_push_ex(*args, C.c_void_p(None), C.c_void_p(ws.data_ptr()), wb, C.c_void_p(st))
            else:
                rc = lib.gast_stream_push(*args, C.c_void_p(ws.data_ptr()), wb, C.c_void_p(st))
            assert rc == 0
            ys.append(y)
        outs.append(torch.stack(ys).cpu())
    assert torch.equal(outs[0], outs[1])
    nc = D.module(Case(case.J, case.fw, case.ch, n, 1, 0, (), case.seed, False, False)).cuda()
    hn = engine.model_handle(nc, dev)
    hn.refresh(nc, st)
    assert lib.gast_stream_state_bytes(hn.h, n) == nb and lib.gast_stream_workspace_bytes(hn.h, n) == wb
    assert lib.gast_stream_latency(hn.h) == (S.receptive_field(case.fw) - 1) // 2
    state = torch.empty(nb, dtype=torch.uint8, device=dev)
    ws = torch.empty(wb, dtype=torch.uint8, device=dev)
    y = torch.empty((n, case.J, 3), device=dev)
    args = [hn.h, C.c_void_p(state.data_ptr()), C.c_int64(0), C.c_void_p(x[0].data_ptr()), C.c_void_p(y.data_ptr()),
            n, C.c_void_p(fresh.data_ptr())]
    assert lib.gast_stream_push(*args, C.c_void_p(ws.data_ptr()), wb, C.c_void_p(st)) != 0
    assert lib.gast_stream_push_ex(*args, C.c_void_p(None), C.c_void_p(ws.data_ptr()), wb, C.c_void_p(st)) == 0
    torch.cuda.synchronize()


def test_weight_change_raises_until_reset():
    case = Case(17, (3, 3, 3), 32, 4, 30, 0, (), 11, False, True)
    m = D.module(case).cuda()
    x = torch.from_numpy(D.frames(case)).cuda()
    ps = PoseStream(m, case.n, augment=True)
    for t in range(6):
        ps.push(x[t])
    X._change('load_state_dict', m, S.Case(17, (3, 3, 3), 32, 4, 30, 0, (), 11))
    with pytest.raises(engine.GastError, match='reset'):
        ps.push(x[6])
    ps.reset([0, 1])
    with pytest.raises(engine.GastError, match='reset'):
        ps.push(x[6])
    ps.end([2, 3])                        # their tails would still be computed from the old-weight history
    with pytest.raises(engine.GastError, match='reset'):
        ps.push(x[6])
    ps.reset()
    y, idx = ps.push(x[6])
    assert idx.tolist() == [-1] * case.n and ps.last_launches > 0


def test_refusals():
    from model.gast_net import SpatioTemporalModel
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    dense = SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], channels=16, dense=True).cuda().eval()
    with pytest.raises(engine.GastError, match='dense'):
        PoseStream(dense, 2)
    m16 = D.module(Case(16, (3, 3, 3), 16, 1, 1, 0, (), 1, False, False)).cuda()
    with pytest.raises(engine.GastError, match='joints'):
        PoseStream(m16, 2, augment=True)
    PoseStream(m16, 2, augment=True, **lists(16)).push(torch.zeros(2, 16, 2, device='cuda'))
    with pytest.raises(RuntimeError, match='causal'):
        CausalStream(m16, 2)


def test_launches_do_not_depend_on_n_and_augment_adds_two():
    case = Case(17, (3, 3, 3), 128, 1, 1, 0, (), 9, False, False)
    m = D.module(case).cuda()
    counts = {}
    for n in (1, 64):
        for aug in (False, True):
            ps = PoseStream(m, n, augment=aug)
            x = torch.zeros(n, 17, 2, device='cuda')
            for _ in range(3):
                ps.push(x)                  # pushes without a fresh or held stream
            counts[n, aug] = ps.last_launches
    assert counts[1, False] == counts[64, False] and counts[1, True] == counts[64, True], counts
    assert counts[1, True] == counts[1, False] + 2, counts
