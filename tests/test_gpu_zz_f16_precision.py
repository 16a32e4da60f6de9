"""GPU: the fp16 inference precision of float32 models (`engine.set_precision(model, 'fp16')`, C ABI
gast_set_precision(h, 16)): the half form's arithmetic and fp16 activations behind float32 input, parameters and
poses, and fp16 stream rings.

  * tied to the half model bit for bit: with fp16-exact weights and input, the 'fp16' forward rounded to fp16 is the
    `model.half()` forward, across schedules, joint counts and widths;
  * whole models against fp64 of the float32 model at TF32's documented bar, over the half tests' matrix;
  * every GEMM launch of 'fp16' forwards and of single-push, chunk and peek stream calls (the tap-rotated weights of
    gast_stream_push_ex included) against fp64 of its own fp16 operands (tests/gemmaudit_half.py);
  * streams: the delayed-stream matrix (causal and not, with and without augment, resets and ends) and chunked pushes
    against fp64; lift_sequences equals tta.evaluate_sequence, a subset listing every stream equals the lockstep
    chunk, peek_subset equals peek, a graphed tick equals the eager calls, a peek leaves the state alone, and the state
    holds the float32 input history and fp16 rings;
  * moving streams: fp16 -> fp16 continues bit for bit, fp16 <-> fp32 within the stream bars; a precision switch on a
    live pool raises and launches nothing, with every stream restarting it reallocates;
  * the refusals, with launch counts, and the round trip to 'fp32'.
Measured errors go to $GAST_TEST_REPORT_DIR/f16_precision.txt when that is set.
"""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth, tta
from gast_b200.realtime import CausalStream, GraphedPoseStream, PoseStream, lift_sequences
from oracle import gast_oracle as O
import delayedref as D
import gemmaudit_half as GAH
import tf32ref as R
import test_gpu_zz_delayed_stream as DS

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')

EXACT_BAR = 5e-3      # max |y - y64| / max |y64|: TF32's documented bar (DESIGN.md §4.1), for forwards and streams
KL, KR = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]


def report(line):
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        with open(os.path.join(REPORT_DIR, 'f16_precision.txt'), 'a') as f:
            f.write(line + '\n')


@pytest.fixture(autouse=True)
def _fp32_core():
    engine.set_gemm_core(0)
    yield
    engine.set_gemm_core(0)


def _adj(J):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))


def _masks(J):
    return O.local_masks(O.adj_from_parents(synth.skeleton_parents(J)))


def _handle(m):
    return list(m.__dict__['_gast_handles'].values())[0]


def _launches(m):
    h = _handle(m)
    return int(h.lib.gast_last_launch_count(h.h))


def _model(J, fw, ch, strided=False, causal=False, dense=False, seed=11):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    if strided:
        m = SpatioTemporalModelOptimized1f(_adj(J), J, 2, J, list(fw), causal=causal, dropout=0.05, channels=ch)
    else:
        m = SpatioTemporalModel(_adj(J), J, 2, J, list(fw), causal=causal, dropout=0.05, channels=ch, dense=dense)
    synth.randomize_module(m, seed)
    return m.eval()


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def _seq(J, T, seed):
    return synth.synth_input(1, T, J, 2, seed=seed)[0]


# ------------------------------------------------------------------------------------------------------------------
# the forward
# ------------------------------------------------------------------------------------------------------------------
MODELS = [  # J, filter widths, channels, strided, causal, dense, B, T  (the half model tests' matrix)
    (17, (3, 3, 3), 128, False, False, False, 6, 40),
    (17, (3, 3, 3), 128, True, False, False, 64, 27),
    (17, (3, 3, 3), 32, False, True, False, 5, 33),
    (17, (3, 3, 3), 64, False, False, True, 4, 31),
    (17, (3, 3, 3, 3), 64, False, False, False, 3, 90),
    (17, (3, 3, 3, 3, 3), 32, True, False, False, 4, 243),
    (15, (3, 3, 3), 64, False, False, False, 5, 30),
    (16, (3, 3, 3), 32, True, True, False, 9, 27),
    (19, (3, 3, 3), 96, False, False, False, 3, 29),
]


@pytest.mark.parametrize('J,fw,ch,strided,causal,dense,B,T', MODELS)
def test_fp16_precision_is_the_half_model_bit_for_bit(J, fw, ch, strided, causal, dense, B, T):
    """fp16-exact weights and input: folding, the weight copy, every GEMM, expand, the row dots, the mix and shrink
    are the half model's arithmetic, and its one output rounding is the only difference"""
    m = _model(J, fw, ch, strided, causal, dense).cuda()
    m.half().float()
    mh = copy.deepcopy(m).half()
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=7 + B)).half()
    engine.set_precision(m, 'fp16')
    with torch.no_grad():
        yh = mh(x.cuda())
        y = m(x.float().cuda())
    assert y.dtype == torch.float32 and yh.dtype == torch.float16
    assert _launches(m) == _launches(mh)
    assert torch.equal(y.half(), yh)


@pytest.mark.parametrize('J,fw,ch,strided,causal,dense,B,T', MODELS)
def test_fp16_precision_against_fp64(J, fw, ch, strided, causal, dense, B, T):
    m = _model(J, fw, ch, strided, causal, dense)
    p = {k: v.numpy() for k, v in m.state_dict().items()}
    x = synth.synth_input(B, T, J, 2, seed=7 + B)
    sched_strided = strided or (T == m.receptive_field() and not dense)
    y64, _ = R.forward(x, p, _masks(J), fw, causal, sched_strided, dense, rnd=False)
    m = m.cuda()
    with torch.no_grad():
        y32 = m(torch.from_numpy(x).cuda()).cpu().numpy()
        engine.set_precision(m, 'fp16')
        y = m(torch.from_numpy(x).cuda())
        assert torch.equal(m(torch.from_numpy(x).cuda()), y)                    # repeatable
    h = _handle(m)
    assert int(h.lib.gast_last_tc_launch_count(h.h)) > 0
    y = y.cpu().numpy()
    e, e32 = _rel(y, y64), _rel(y, y32)
    report('model J%d fw%s c%d strided %d causal %d dense %d B%d T%d: max|y - y64| / max|y64| %.2e, from fp32 grade '
           '%.2e' % (J, fw, ch, strided, causal, dense, B, T, e, e32))
    assert e < EXACT_BAR, e


def test_fp16_mpjpe_chunked_and_profile():
    m = engine.set_precision(_model(17, (3, 3, 3), 64).cuda(), 'fp16')
    x = torch.from_numpy(synth.synth_input(5, 60, 17, 2, seed=3)).cuda()
    with torch.no_grad():
        y = m(x)
        y2, loss = engine.run_model_mpjpe(m, x, torch.zeros_like(y))
        yc = engine.run_model_chunked(m, x, 10 ** 6)
        yw = engine.run_model_chunked(m, x, 7)
    assert y.dtype == torch.float32
    assert torch.equal(y, y2) and torch.equal(y, yc)                            # one pass: the same launches
    assert abs(float(loss) - float(y.double().norm(dim=-1).mean())) < 1e-5 * float(loss)
    assert _rel(yw.cpu(), y.cpu()) < 2 * EXACT_BAR                              # other tiles: other roundings
    assert engine.profile_forward(m, x, reps=1)['gemm_core'].startswith('wgmma-fp16')


def test_fp16_then_fp32_gives_the_fp32_bits_back():
    m = _model(17, (3, 3, 3), 64).cuda()
    xs = [torch.from_numpy(synth.synth_input(6, T, 17, 2, seed=T)).cuda() for T in (27, 40)]

    def run():
        with torch.no_grad():
            return [m(x) for x in xs], m._gast_last_launches

    a, la = run()
    engine.set_precision(m, 'fp16')
    h, lh = run()
    engine.set_precision(m, 'fp32')
    b, lb = run()
    for u, v, w in zip(a, h, b):
        assert torch.equal(u, w)
        assert _rel(v.cpu(), u.cpu()) > 1e-5                                    # fp16 differs from fp32 grade
    assert la == lh == lb


# ------------------------------------------------------------------------------------------------------------------
# every GEMM launch of 'fp16' forwards and stream calls, audited
# ------------------------------------------------------------------------------------------------------------------
def _audited(m, fn):
    h = _handle(m)
    aud = GAH.Auditor()
    aud.install(h.lib, h.h)
    try:
        try:
            out = fn()
        except engine.GastError as ex:
            raise AssertionError('%s\n%s' % (ex, aud.failure)) from ex
    finally:
        h.lib.gast_debug_set_gemm_audit(h.h, _lib.GemmAuditFn(), None)
    assert aud.failure is None, aud.failure
    assert aud.records
    return out, aud.records


@pytest.mark.parametrize('J,fw,ch,strided,causal,B,T', [
    (17, (3, 3, 3), 64, False, False, 3, 33),      # dilated taps: gathered segments, residuals, SemCH, attention mix
    (17, (3, 3, 3), 32, True, True, 4, 27),        # strided, causal
])
def test_every_gemm_of_an_fp16_forward_against_fp64(J, fw, ch, strided, causal, B, T):
    m = engine.set_precision(_model(J, fw, ch, strided, causal).cuda(), 'fp16')
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=3)).cuda()
    with torch.no_grad():
        y = m(x)
        ya, recs = _audited(m, lambda: m(x))
    h = _handle(m)
    assert len(recs) == int(h.lib.gast_last_tc_launch_count(h.h))
    assert torch.equal(ya, y)
    assert {r['epi'] for r in recs} == {'plain', 'semch'}
    if not strided:
        assert any(r['tma_mask'] != (1 << r['nseg']) - 1 for r in recs)         # a gathered tap segment
    report('audit forward J%d c%d strided %d: %d launches, worst/bound %.3f'
           % (J, ch, strided, len(recs), max(r['worst'] for r in recs)))


@pytest.mark.parametrize('causal', [True, False])
def test_every_gemm_of_fp16_stream_calls_against_fp64(causal):
    J, n = 17, 3
    m = engine.set_precision(_model(J, (3, 3, 3), 64, causal=causal).cuda(), 'fp16')
    frames = torch.from_numpy(synth.synth_input(n, 40, J, 2, seed=J)).cuda()
    ps = PoseStream(m, n)
    with torch.no_grad():
        for t in range(29):                                                    # the 27-slot ring wraps
            ps.push(frames[:, t])
        _, single = _audited(m, lambda: ps.push(frames[:, 29]))                 # gast_stream_push_ex: rotated taps
        _, chunk = _audited(m, lambda: ps.push_frames(frames[:, 30:36].contiguous()))
        _, subset = _audited(m, lambda: ps.push(frames[[0, 2], 36], streams=[0, 2]))
        peek = _audited(m, lambda: ps.peek(4))[1] if not causal else []
    recs = single + chunk + subset + peek
    assert any(r['tma_mask'] != (1 << r['nseg']) - 1 for r in single)          # the ring's tap slots, gathered
    report('audit streams causal %d: %d launches, worst/bound %.3f' % (causal, len(recs), max(r['worst'] for r in recs)))


# ------------------------------------------------------------------------------------------------------------------
# streams against fp64
# ------------------------------------------------------------------------------------------------------------------
STREAM_CASES = ['j17_333_c128_n37_aug', 'j17_333_c64_causal_n6_aug', 'j16_353_c32_n16']


@pytest.mark.parametrize('name', STREAM_CASES)
def test_delayed_stream_matrix_against_fp64(name):
    case = DS.CASES[name]
    m = engine.set_precision(D.module(case).cuda(), 'fp16')
    got, idx, ps = DS.push_all(case, m)
    assert ps._ring == 'fp16'
    for s in range(case.n):
        assert np.array_equal(idx[s], D.expected_index(case, s)), s
    picked = DS.sample(case)
    ref, ridx = D.reference(case, picked)
    mx, l2 = D.errors(got[list(picked)], ref, ridx)
    report('delayed %s: max %.2e, L2 %.2e' % (name, mx, l2))
    assert mx < EXACT_BAR, mx


def _stream_poses(ps, seq, pushes):
    """push `seq` (T, J, 2) on stream 0 of a 2-stream pool (stream 1 gets the reversed sequence) by `pushes` (chunk
    lengths, 1 = a single push), end it and flush -> the poses (T, J, 3) of stream 0"""
    T = seq.shape[0]
    both = np.stack([seq, seq[::-1].copy()])
    got, t = {}, 0
    for K in pushes + [1] * (T + ps.latency):
        if t >= T + ps.latency:
            break
        if t == T:
            ps.end()
        if t < T and K > 1:
            K = min(K, T - t)
            y, idx = ps.push_frames(torch.from_numpy(both[:, t:t + K].copy()).cuda())
            for k in range(K):
                if idx[0, k] >= 0:
                    got[int(idx[0, k])] = y[0, k].cpu().numpy()
        else:
            y, idx = ps.push(torch.from_numpy(both[:, min(t, T - 1)].copy()).cuda())
            if idx[0] >= 0:
                got[int(idx[0])] = y[0].cpu().numpy()
            K = 1
        t += K
    return np.stack([got[i] for i in range(T)])


@pytest.mark.parametrize('causal,augment', [(False, True), (True, False)])
def test_single_and_chunked_pushes_against_fp64(causal, augment):
    fw = (3, 3, 3)
    m = _model(17, fw, 64, causal=causal)
    seq = _seq(17, 60, 5)
    ref = D.sequence_poses([seq], 17, fw, causal, augment, D.symmetry(17), m.state_dict())[0]
    engine.set_precision(m.cuda(), 'fp16')
    single = _stream_poses(PoseStream(m, 2, augment=augment), seq, [])
    chunked = _stream_poses(PoseStream(m, 2, augment=augment), seq, [7, 1, 30, 2])
    e1, e2 = _rel(single, ref), _rel(chunked, ref)
    report('pushes causal %d augment %d against fp64: single %.2e, chunks %.2e' % (causal, augment, e1, e2))
    assert e1 < EXACT_BAR and e2 < EXACT_BAR


# ------------------------------------------------------------------------------------------------------------------
# streams: exact equalities and the state
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fw,ch,causal', [((3, 3, 3), 128, False), ((3, 3, 3), 64, True)])
def test_lift_sequences_equals_evaluate_sequence(fw, ch, causal):
    m = engine.set_precision(_model(17, fw, ch, causal=causal).cuda(), 'fp16')
    seqs = [_seq(17, L, 100 + L) for L in (70, 5, 33, 90)]
    out = lift_sequences(m, seqs, n_streams=2, chunk=24, augment=True)
    for k, sq in enumerate(seqs):
        want = tta.evaluate_sequence(m, sq, KL, KR, KL, KR, causal=causal)
        assert torch.equal(out[k], want), k


def test_subset_peek_and_state_equalities():
    m = engine.set_precision(_model(17, (3, 3, 3), 64).cuda(), 'fp16')
    n, K = 5, 6
    x = torch.from_numpy(synth.synth_input(n, 3 * K, 17, 2, seed=8)).cuda()
    a, b = PoseStream(m, n), PoseStream(m, n)
    rev = list(range(n))[::-1]
    for c in range(3):
        xa = x[:, c * K:(c + 1) * K].contiguous()
        ya, ia = a.push_frames(xa)                                              # lockstep chunk
        yb, ib = b.push_frames(xa[rev].contiguous(), streams=rev)               # a subset listing every stream
        assert torch.equal(yb, ya[rev]) and torch.equal(ib, ia[rev])
    assert torch.equal(a._state, b._state)
    before = a._state.clone()
    pa, qa = a.peek()
    pb, qb = a.peek(streams=rev)
    assert torch.equal(pb, pa[rev]) and torch.equal(qb, qa[rev])
    assert torch.equal(a._state, before)                                        # a peek writes no state


def test_graphed_tick_equals_eager_calls():
    m = engine.set_precision(_model(17, (3, 3, 3), 64).cuda(), 'fp16')
    n, K, P = 3, 4, 5
    g = GraphedPoseStream(m, n, augment=True, K=K, peek=P)
    e = PoseStream(m, n, augment=True)
    x = torch.from_numpy(synth.synth_input(n, 5 * K, 17, 2, seed=4)).cuda()
    for c in range(5):
        xc = x[:, c * K:(c + 1) * K].contiguous()
        y, idx, py, pidx = g.push(xc)
        ye, ie = e.push_frames(xc)
        pe, pie = e.peek(P)
        assert torch.equal(idx, ie) and torch.equal(pidx, pie)
        assert torch.equal(y[idx >= 0], ye[ie >= 0]) and torch.equal(py[pidx >= 0], pe[pie >= 0])


def _state_bytes(J, F, fw, ch, n, ring_esize):
    al = lambda b: (b + 255) // 256 * 256                                      # noqa: E731
    total, d = al(n * fw[0] * J * F * 4), fw[0]
    for i in range(1, len(fw)):
        total += al(fw[i] * d * n * J * (ch << i) * ring_esize)
        d *= fw[i]
    return total + 256


@pytest.mark.parametrize('fw,ch,n', [((3, 3, 3), 128, 7), ((3, 5, 3), 32, 3), ((3, 3, 3, 3, 3), 64, 1)])
def test_state_holds_float32_history_and_fp16_rings(fw, ch, n):
    m = _model(17, fw, ch).cuda()
    with torch.no_grad():
        m(torch.from_numpy(synth.synth_input(1, m.receptive_field(), 17, 2, seed=1)).cuda())
    h = _handle(m)
    assert h.lib.gast_stream_state_bytes(h.h, n) == _state_bytes(17, 2, fw, ch, n, 4)
    engine.set_precision(m, 'fp16')
    h.apply_core(m)
    assert h.lib.gast_stream_state_bytes(h.h, n) == _state_bytes(17, 2, fw, ch, n, 2)
    engine.set_precision(m, 'fp32')
    h.apply_core(m)


# ------------------------------------------------------------------------------------------------------------------
# moving streams and switching precision
# ------------------------------------------------------------------------------------------------------------------
def _causal_setup(T=60):
    fw = (3, 3, 3)
    m = _model(17, fw, 64, causal=True)
    seqs = [_seq(17, T, 21), _seq(17, T, 22)]
    ref = np.stack(D.sequence_poses(seqs, 17, fw, True, False, D.symmetry(17), m.state_dict()))
    x = torch.from_numpy(np.stack(seqs)).cuda()                                # (2, T, J, 2)
    return m.cuda(), x, ref


def test_fp16_pool_moves_bit_for_bit():
    m, x, _ = _causal_setup()
    engine.set_precision(m, 'fp16')
    a = PoseStream(m, 2)
    a.push_frames(x[:, :20].contiguous())
    snap = a.export_streams([0, 1])
    b = PoseStream(m, 4)
    b.import_streams(snap, [3, 1])
    ya, _ = a.push_frames(x[:, 20:35].contiguous())
    yb, _ = b.push_frames(x[:, 20:35].contiguous(), streams=[3, 1])
    assert torch.equal(ya, yb)


@pytest.mark.parametrize('src,dst', [('fp16', 'fp32'), ('fp32', 'fp16')])
def test_streams_move_between_precisions(src, dst):
    m, x, ref = _causal_setup()
    engine.set_precision(m, src)
    a = PoseStream(m, 2)
    y0, _ = a.push_frames(x[:, :20].contiguous())
    snap = a.export_streams([0, 1])
    engine.set_precision(m, dst)
    b = PoseStream(m, 2)
    b.import_streams(snap, [0, 1])
    assert b._ring == ('fp16' if dst == 'fp16' else 'fp32')
    y1, _ = b.push_frames(x[:, 20:].contiguous())
    e0, e1 = _rel(y0.cpu(), ref[:, :20]), _rel(y1.cpu(), ref[:, 20:])
    report('move %s -> %s: before %.2e, after %.2e' % (src, dst, e0, e1))
    assert e0 < EXACT_BAR and e1 < EXACT_BAR
    engine.set_precision(m, 'fp32')


def test_precision_switch_on_a_live_pool():
    m, x, ref = _causal_setup()
    ps = CausalStream(m, 2)
    ps.push_frames(x[:, :10].contiguous())
    engine.set_precision(m, 'tf32')                                           # the same ring type: kept
    ps.push(x[:, 10])
    n0 = _launches(m)
    assert n0 > 0 and ps._ring == 'fp32'
    engine.set_precision(m, 'fp16')
    with pytest.raises(engine.GastError, match='export_streams'):
        ps.push(x[:, 11])
    assert _launches(m) == n0                                                 # refused before the call's first launch
    state = ps._state
    ps.reset()                                                                # every stream restarts: reallocated
    y = ps.push_frames(x[:, :30].contiguous())
    assert ps._ring == 'fp16' and ps._state is not state and ps._state.numel() < state.numel()
    assert _rel(y.cpu(), ref[:, :30]) < EXACT_BAR
    engine.set_precision(m, 'fp32')
    with pytest.raises(engine.GastError, match='export_streams'):
        ps.push(x[:, 30])
    g = GraphedPoseStream(m, 2, K=2)
    g.push(x[:, :2].contiguous())
    engine.set_precision(m, 'fp16')
    with pytest.raises(engine.GastError, match='set_precision'):
        g.push(x[:, 2:4].contiguous())                                        # a switch since the capture
    engine.set_precision(m, 'fp32')


def test_streams_round_trip_after_restart():
    T = 27                                   # R_max of the 3-3-3 model: every restart lands on the same ring phases
    m, x, _ = _causal_setup(T)
    ps = CausalStream(m, 2)
    y32 = torch.stack([ps.push(x[:, t]) for t in range(T)], 1)
    engine.set_precision(m, 'fp16')
    ps.reset()
    y16 = torch.stack([ps.push(x[:, t]) for t in range(T)], 1)
    assert ps._ring == 'fp16'
    engine.set_precision(m, 'fp32')
    ps.reset()
    yb = torch.stack([ps.push(x[:, t]) for t in range(T)], 1)
    assert torch.equal(yb, y32)
    assert 1e-5 < _rel(y16.cpu(), y32.cpu()) < EXACT_BAR


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
def test_library_refusals():
    m = _model(17, (3, 3, 3), 32).cuda()
    x = torch.from_numpy(synth.synth_input(2, 27, 17, 2, seed=1)).cuda()
    with torch.no_grad():
        m(x)
    h = _handle(m)
    lib = h.lib
    n0 = _launches(m)
    assert lib.gast_set_precision(h.h, 2) != 0 and 'mode' in _lib.last_error()
    assert lib.gast_set_gemm_core(h.h, 1) == 0                                 # FFMA first, then fp16
    assert lib.gast_set_precision(h.h, 16) != 0 and 'tensor-core' in _lib.last_error()
    assert lib.gast_set_gemm_core(h.h, 0) == 0
    assert lib.gast_set_precision(h.h, 16) == 0                                # fp16 first, then FFMA
    assert lib.gast_set_gemm_core(h.h, 1) != 0 and 'fp16' in _lib.last_error()
    assert lib.gast_set_activation_dtype(h.h, 1) != 0 and 'precision is 16' in _lib.last_error()
    assert lib.gast_train_workspace_bytes(h.h, 2, 27, C.c_float(0.0)) == 0
    assert 'inference-only' in _lib.last_error()
    assert lib.gast_eval_backward_workspace_bytes(h.h, 2, 27, 1) == 0
    assert 'inference-only' in _lib.last_error()
    assert lib.gast_set_precision(h.h, 0) == 0
    assert _launches(m) == n0
    h.precision = 0

    mh = _model(17, (3, 3, 3), 32).cuda().half()
    with torch.no_grad():
        mh(x.half())
    hh = _handle(mh)
    assert hh.lib.gast_set_precision(hh.h, 16) != 0 and 'fp16' in _lib.last_error()

    J = 24                                                                     # the C ABI: more joints than half takes
    eye = torch.eye(J)
    chain = eye + torch.diag(torch.ones(J - 1), 1) + torch.diag(torch.ones(J - 1), -1)
    hj = engine._Handle(None, _lib.KIND_MODEL, torch.device('cuda', 0), dict(
        num_joints=J, in_features=2, channels=32, filter_widths=[3, 3], causal=0, dense=0, strided=0, heads=4),
        sym=eye, con=chain)
    assert hj.lib.gast_set_precision(hj.h, 16) != 0 and 'at most 20 joints' in _lib.last_error()
    assert hj.lib.gast_set_precision(hj.h, 1) == 0


def test_engine_refusals():
    x = torch.from_numpy(synth.synth_input(2, 27, 17, 2, seed=2)).cuda()
    mw = engine.set_precision(_model(17, (3, 3, 3), 48).cuda(), 'fp16')       # widths the half form does not take
    with pytest.raises(engine.GastError, match='multiple of 32'):
        with torch.no_grad():
            mw(x)
    assert _launches(mw) == 0

    mh = _model(17, (3, 3, 3), 32).cuda().half()
    with torch.no_grad():
        mh(x.half())
    n0 = _launches(mh)
    engine.set_precision(mh, 'fp16')
    with pytest.raises(engine.GastError, match=r"set_precision\(model, 'fp32'\)"):
        with torch.no_grad():
            mh(x.half())
    assert _launches(mh) == n0
    engine.set_precision(mh, 'fp32')
    with torch.no_grad():
        mh(x.half())

    m = engine.set_precision(_model(17, (3, 3, 3), 32).cuda(), 'fp16')
    with torch.no_grad():
        m(x)
    n0 = _launches(m)
    with pytest.raises(engine.GastError, match=r"set_precision\(model, 'fp32'\)"):
        m.train()(x)
    m.eval()
    with pytest.raises(engine.GastError, match=r"set_precision\(model, 'fp32'\)"):
        m(x.clone().requires_grad_(True))
    with pytest.raises(engine.GastError, match=r"set_precision\(model, 'fp32'\)"):
        m(x)                                                                   # parameters require grad
    assert _launches(m) == n0
    with pytest.raises(engine.GastError, match="'fp16'"):
        engine.set_training_precision(m, 'fp16')

    # with the training precision at TF32, training and gradients run at 'fp16' as they do at 'tf32'
    engine.set_training_precision(m, 'tf32')
    m.train()
    m(x).abs().mean().backward()
    assert all(p.grad is not None for p in m.parameters() if p.requires_grad)
    m.eval()
    for p in m.parameters():
        p.grad = None
    y = m(x)
    with torch.no_grad():
        assert torch.equal(y.detach(), m(x))                                  # the 'fp16' inference forward
    y.abs().mean().backward()
    assert all(p.grad is not None for p in m.parameters() if p.requires_grad)
