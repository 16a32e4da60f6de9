"""GPU: half-precision models (`model.half()`, the library's gast_set_activation_dtype(h, GAST_F16)).

  * gast_debug_gemm with tc_mode 16: the half form of the wgmma core (fp16 A and W from shared memory, fp32
    accumulation, fp16 output) against fp64 of the same fp16 operands, across N, K and ring phases.
  * every GEMM launch of half forwards (tests/gemmaudit_half.py) against fp64 of its own fp16 operands: the plain and
    SemCH epilogues, TMA-fed and gathered (tap) segments, residuals.  (The half form has no fused-attention epilogue:
    more than 20 joints are refused in half, and the model classes take at most 19.)
  * whole half models across joint counts, schedules (dilated, strided, causal, dense), depths and widths against
    fp64 of the same fp16-exact weights and input, at TF32's documented bar (DESIGN.md §4.1).
  * the chunked forward equals the whole forward bit for bit when one pass covers the call; calls repeat bit for bit.
  * model.half() then model.float() gives the fp32 forward's bits back.
  * the refusals: training, autograd, run_model_mpjpe, the streams, lift_sequences, tta.evaluate_sequence,
    sub-modules, mixed dtypes, and the bind check of non-float32 tensors.
Measured errors go to $GAST_TEST_REPORT_DIR/half.txt when that is set.
"""
import os

import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth, tta
import gemmaudit as GA
import gemmaudit_half as GAH
from gast_b200.realtime import CausalStream, PoseStream, lift_sequences
from oracle import gast_oracle as O
import tf32ref as R

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')

EXACT_BAR = 5e-3      # max |y - y64| / max |y64| of a half model: TF32's documented bar (DESIGN.md §4.1)
F16_ULP = 2.0 ** -11  # one fp16 rounding of the output, relative
ACC_BAR = 1e-5        # fp32 accumulation (chained k16 MMAs) relative to sum |a| |w|


def report(line):
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        with open(os.path.join(REPORT_DIR, 'half.txt'), 'a') as f:
            f.write(line + '\n')


def _adj(J):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))


def _masks(J):
    return O.local_masks(O.adj_from_parents(synth.skeleton_parents(J)))


def _handle(m):
    return list(m.__dict__['_gast_handles'].values())[0]


def _model(J, fw, ch, strided=False, causal=False, dense=False, seed=11):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    if strided:
        m = SpatioTemporalModelOptimized1f(_adj(J), J, 2, J, list(fw), causal=causal, dropout=0.05, channels=ch)
    else:
        m = SpatioTemporalModel(_adj(J), J, 2, J, list(fw), causal=causal, dropout=0.05, channels=ch, dense=dense)
    synth.randomize_module(m, seed)
    return m.eval()


# ------------------------------------------------------------------------------------------------------------------
# one GEMM of the half form (gast_debug_gemm, tc_mode 16)
# ------------------------------------------------------------------------------------------------------------------
def _gemm_h(a, w, M, N, K):
    lib = _lib.load()
    o = torch.full((M, N), float('nan'), dtype=torch.float16, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, 16, 0, None,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return o.float().cpu().numpy().astype(np.float64)


# K / 32 stages: fewer than the 6 ring slots, full, one wrap, many; N: partial, one and several column tiles
@pytest.mark.parametrize('K', [32, 64, 192, 224, 512, 1536])
@pytest.mark.parametrize('N', [96, 128, 384])
@pytest.mark.parametrize('wscale', [1.0, 300.0])
def test_half_gemm_against_fp64_of_its_operands(K, N, wscale):
    M = 1000 + K // 32                                   # a partial last row tile
    g = torch.Generator().manual_seed(K * 7 + N)
    a = torch.randn(M, K, generator=g).half()
    w = (torch.randn(N, K, generator=g) * 0.05 * wscale).half().float()   # fp16-exact, as a half model's weights
    out = _gemm_h(a.cuda(), w.cuda(), M, N, K)
    a64, w64 = a.double().numpy(), w.double().numpy()
    ref = a64 @ w64.T
    mag = np.abs(a64) @ np.abs(w64).T
    err = np.abs(out - ref)
    bound = F16_ULP * np.abs(ref) + ACC_BAR * mag + 1e-30
    report('gemm M%d N%d K%d wscale %g: max err / bound %.3f, max rel %.2e'
           % (M, N, K, wscale, float((err / bound).max()), float(err.max() / np.abs(ref).max())))
    assert np.isfinite(out).all()
    assert (err <= bound).all(), float((err / bound).max())
    assert np.array_equal(out, _gemm_h(a.cuda(), w.cuda(), M, N, K))          # repeatable


def test_half_gemm_refuses_shapes_it_does_not_take():
    lib = _lib.load()
    a = torch.zeros(64, 48, dtype=torch.float16, device='cuda')
    w = torch.zeros(32, 48, device='cuda')
    o = torch.zeros(64, 32, dtype=torch.float16, device='cuda')
    assert lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), 64, 32, 48, 0, 16, 0, None,
                               torch.cuda.current_stream().cuda_stream) != 0       # K % 32 != 0
    assert 'not supported' in _lib.last_error()


# ------------------------------------------------------------------------------------------------------------------
# whole models
# ------------------------------------------------------------------------------------------------------------------
MODELS = [  # J, filter widths, channels, strided, causal, dense, B, T
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


def _half_case(J, fw, ch, strided, causal, dense, B, T):
    m = _model(J, fw, ch, strided, causal, dense).cuda().half()
    p = {k: v.double().cpu().numpy() if v.is_floating_point() else v.cpu().numpy() for k, v in m.state_dict().items()}
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=7 + B)).half()
    sched_strided = strided or (T == m.receptive_field() and not dense)
    y64, _ = R.forward(x.double().numpy(), p, _masks(J), fw, causal, sched_strided, dense, rnd=False)
    with torch.no_grad():
        y = m(x.cuda())
    return m, x, y, y64


@pytest.mark.parametrize('J,fw,ch,strided,causal,dense,B,T', MODELS)
def test_half_model_against_fp64(J, fw, ch, strided, causal, dense, B, T):
    m, x, y, y64 = _half_case(J, fw, ch, strided, causal, dense, B, T)
    assert y.dtype == torch.float16 and tuple(y.shape) == y64.shape
    h = _handle(m)
    assert int(h.lib.gast_last_tc_launch_count(h.h)) > 0
    yf = y.float().cpu().numpy().astype(np.float64)
    e = float(np.abs(yf - y64).max() / np.abs(y64).max())
    report('model J%d fw%s c%d strided %d causal %d dense %d B%d T%d: max|y - y64| / max|y64| %.2e'
           % (J, fw, ch, strided, causal, dense, B, T, e))
    assert e < EXACT_BAR, e
    with torch.no_grad():
        assert torch.equal(m(x.cuda()), y)                                      # repeatable


# ------------------------------------------------------------------------------------------------------------------
# every GEMM launch of a half forward, audited
# ------------------------------------------------------------------------------------------------------------------
AUDITED = [  # J, filter widths, channels, strided, causal, B, T
    (17, (3, 3, 3), 64, False, False, 3, 33),      # dilated taps: gathered segments, residuals, SemCH, attention mix
    (17, (3, 3, 3), 32, True, True, 4, 27),        # strided, causal
]


@pytest.mark.parametrize('J,fw,ch,strided,causal,B,T', AUDITED)
def test_every_gemm_of_a_half_forward_against_fp64(J, fw, ch, strided, causal, B, T):
    m = _model(J, fw, ch, strided, causal).cuda().half()
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=3)).half().cuda()
    with torch.no_grad():
        y = m(x)                                                                # creates the handle
    h = _handle(m)
    aud = GAH.Auditor()
    aud.install(h.lib, h.h)
    try:
        with torch.no_grad():
            try:
                ya = m(x)
            except engine.GastError as ex:
                raise AssertionError('%s\n%s' % (ex, aud.failure)) from ex
    finally:
        h.lib.gast_debug_set_gemm_audit(h.h, _lib.GemmAuditFn(), None)
    assert aud.failure is None, aud.failure
    recs = aud.records
    assert len(recs) == int(h.lib.gast_last_tc_launch_count(h.h)) > 0           # every GEMM launch, all in half
    assert torch.equal(ya, y)                                                   # the audit changes nothing
    epis = {r['epi'] for r in recs}
    assert epis == {'plain', 'semch'}
    assert any(r['tma_mask'] == (1 << r['nseg']) - 1 for r in recs)            # TMA-fed segments
    if not strided:
        assert any(r['tma_mask'] != (1 << r['nseg']) - 1 for r in recs)        # a gathered tap segment
    for r in recs:
        report('audit J%d fw%s c%d strided %d causal %d: launch %d %s N %d K %d tma %d worst/bound %.3f max rel %.2e'
               % (J, fw, ch, strided, causal, r['index'], r['epi'], r['N'], r['K'], r['tma_mask'], r['worst'],
                  r['max_rel']))


def test_half_audit_catches_a_wrong_output():
    """the audit's bound is tight enough to refuse an output moved by a few fp16 ulps"""
    m = _model(17, (3, 3, 3), 32).cuda().half()
    x = torch.from_numpy(synth.synth_input(2, 27, 17, 2, seed=3)).half().cuda()
    with torch.no_grad():
        m(x)
    h = _handle(m)
    aud = GAH.Auditor()
    caught = []
    orig = GAH.check

    def corrupt(P, S, out1):
        out1 = out1.copy()
        out1[0, 0] = np.float32(np.float16(out1[0, 0]) * np.float16(1.01)) + np.float32(0.01)
        try:
            return orig(P, S, out1)
        except GA.AuditError as ex:
            caught.append(str(ex))
            return orig(P, S, GAH.read_out(P, aud.mem))
    GAH.check = corrupt
    aud.install(h.lib, h.h)
    try:
        with torch.no_grad():
            m(x)
    finally:
        GAH.check = orig
        h.lib.gast_debug_set_gemm_audit(h.h, _lib.GemmAuditFn(), None)
    assert aud.failure is None, aud.failure
    assert caught and len(caught) == len(aud.records)


@pytest.mark.parametrize('max_frames', [10 ** 6, 7])
def test_half_chunked_forward(max_frames):
    m = _model(17, (3, 3, 3), 64).cuda().half()
    x = torch.from_numpy(synth.synth_input(5, 60, 17, 2, seed=3)).half().cuda()
    with torch.no_grad():
        y = m(x)
        yc = engine.run_model_chunked(m, x, max_frames)
    assert yc.dtype == torch.float16
    if max_frames >= y.shape[0] * y.shape[1]:
        assert torch.equal(yc, y)                                               # one pass: the same launches
    else:
        d = float((yc.float() - y.float()).abs().max() / y.float().abs().max())
        assert d < 2 * EXACT_BAR, d                                             # other tiles: other roundings
        with torch.no_grad():
            assert torch.equal(engine.run_model_chunked(m, x, max_frames), yc)  # repeatable


def test_half_then_float_gives_the_fp32_bits_back():
    m = _model(17, (3, 3, 3), 64).cuda()
    x = torch.from_numpy(synth.synth_input(4, 40, 17, 2, seed=5)).cuda()
    with torch.no_grad():
        yh = m.half()(x.half())
        y32b = m.float()(x)
    assert yh.dtype == torch.float16 and y32b.dtype == torch.float32
    m2 = _model(17, (3, 3, 3), 64).cuda()
    m2.load_state_dict(m.state_dict())
    with torch.no_grad():
        assert torch.equal(m2(x), y32b)                                         # nothing of half is left over
    h = _handle(m)
    assert h.f32 is None and h.act_dtype == 0


def test_half_rounded_weights_round_trip_bitwise():
    m = _model(17, (3, 3, 3), 64).cuda()
    m.half().float()                                                            # fp16-exact fp32 weights
    x = torch.from_numpy(synth.synth_input(4, 40, 17, 2, seed=5)).cuda()
    with torch.no_grad():
        y32 = m(x)
        m.half()(x.half())
        assert torch.equal(m.float()(x), y32)


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
def _launches(m):
    """the library's launch count of the handle's last call (restarted by every call that gets past its checks)"""
    h = _handle(m)
    return int(h.lib.gast_last_launch_count(h.h))


def test_half_refusals():
    m = _model(17, (3, 3, 3), 32).cuda().half()
    x = torch.from_numpy(synth.synth_input(2, 27, 17, 2, seed=1)).half().cuda()
    with torch.no_grad():
        m(x)
    n0 = _launches(m)
    assert n0 > 0

    with pytest.raises(engine.GastError, match='float32'):
        with torch.no_grad():
            m(x.float())                                                        # fp32 input into a half model
    with pytest.raises(engine.GastError, match='inference only'):
        m(x)                                                                    # would build an autograd graph
    with pytest.raises(engine.GastError, match='inference only'):
        m.train()(x)
    m.eval()
    with pytest.raises(engine.GastError, match='inference only'):
        engine.run_model_mpjpe(m, x, torch.zeros(2, 1, 17, 3, dtype=torch.float16, device='cuda'))
    with pytest.raises(engine.GastError, match='inference only'):
        PoseStream(m, 2)
    with pytest.raises(engine.GastError, match='inference only'):
        CausalStream(_model(17, (3, 3, 3), 32, causal=True).cuda().half(), 2)
    with pytest.raises(engine.GastError, match='inference only'):
        lift_sequences(m, [np.zeros((30, 17, 2), np.float32)])
    with pytest.raises(engine.GastError, match='inference only'):
        tta.evaluate_sequence(m, np.zeros((30, 17, 2), np.float32), [1], [4], [1], [4])
    with pytest.raises(engine.GastError, match='inference only'):
        m.layers_graph_conv[0].local_graph_layer(torch.zeros(2, 1, 17, 32, dtype=torch.float16, device='cuda'))
    with pytest.raises(engine.GastError, match='TF32'):
        with torch.no_grad():
            engine.set_precision(m, 'tf32')(x)
    engine.set_precision(m, 'fp32')
    assert _launches(m) == n0                                                   # nothing launched since

    mw = _model(17, (3, 3, 3), 48).cuda().half()                               # widths the half form does not take
    with pytest.raises(engine.GastError, match='multiple of 32'):
        with torch.no_grad():
            mw(x)
    assert int(_handle(mw).lib.gast_last_launch_count(_handle(mw).h)) == 0     # refused before any launch

    mf = _model(17, (3, 3, 3), 32).cuda()
    with pytest.raises(engine.GastError, match='float16'):
        with torch.no_grad():
            mf(x)                                                               # fp16 input into a float model
    mf.shrink.half()
    with pytest.raises(engine.GastError, match='all be float32 or all float16'):
        with torch.no_grad():
            mf(x.float())                                                       # a module of mixed dtypes


def test_half_library_refusals():
    m = _model(17, (3, 3, 3), 32).cuda().half()
    x = torch.from_numpy(synth.synth_input(2, 27, 17, 2, seed=1)).half().cuda()
    with torch.no_grad():
        m(x)
    h = _handle(m)
    lib = h.lib
    assert lib.gast_set_gemm_core(h.h, 1) != 0 and 'fp16' in _lib.last_error()
    assert lib.gast_set_precision(h.h, 1) != 0 and 'fp16' in _lib.last_error()
    assert lib.gast_train_workspace_bytes(h.h, 2, 27, 0.0) == 0 and 'fp16' in _lib.last_error()
    assert lib.gast_stream_state_bytes(h.h, 2) == 0 and 'fp16' in _lib.last_error()
    assert lib.gast_eval_backward_workspace_bytes(h.h, 2, 27, 0) == 0 and 'fp16' in _lib.last_error()


def test_half_refuses_more_than_20_joints():
    """a MODEL handle of 24 joints (C ABI; the model classes take at most 19) refuses half before any launch"""
    J = 24
    eye = torch.eye(J)
    chain = eye + torch.diag(torch.ones(J - 1), 1) + torch.diag(torch.ones(J - 1), -1)
    h = engine._Handle(None, _lib.KIND_MODEL, torch.device('cuda', 0), dict(
        num_joints=J, in_features=2, channels=32, filter_widths=[3, 3], causal=0, dense=0, strided=0, heads=4),
        sym=eye, con=chain)
    assert h.lib.gast_set_activation_dtype(h.h, 1) != 0
    assert 'at most 20 joints' in _lib.last_error()
    assert h.lib.gast_set_activation_dtype(h.h, 0) == 0


def test_bind_refuses_non_float32_tensors():
    m = _model(17, (3, 3, 3), 32).cuda()
    with torch.no_grad():
        m(torch.from_numpy(synth.synth_input(2, 27, 17, 2, seed=1)).cuda())
    h = _handle(m)
    n0 = int(h.lib.gast_last_launch_count(h.h))
    with pytest.raises(engine.GastError, match="'w' is torch.float16"):
        engine._bind(h, 'gast_bind', [('w', torch.zeros(8, dtype=torch.float16, device='cuda'))])
    with pytest.raises(engine.GastError, match="'w' is torch.bfloat16"):
        engine._bind(h, 'gast_bind', [('w', torch.zeros(8, dtype=torch.bfloat16, device='cuda'))])
    assert int(h.lib.gast_last_launch_count(h.h)) == n0
