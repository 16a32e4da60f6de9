"""GPU: the batched inference forward and every attention-kernel variant the drop-in modules reach, against fp64.

The reference is the torch-CPU port (oracle/gast_torch_ref.py) in float64 (tests/fp64ref.py).  Every case is held
to two fp32-grade bars, max |y - y64| / max |y64| and the relative L2 error, on both GEMM cores, and asserts the
kernel path it targets through the launch kinds of the module's own handle (engine.LAUNCH_KINDS), so that a case
that falls back to the other core does not pass as a check of it.

  * Sub-modules: MultiGlobalGraph with 1, 3 and 4 heads at J = 17, 19 and 24 (tensor-core `g` GEMM + global_mix up
    to J = 20, the fused tensor-core EPI_GLOBAL epilogue with hpt = heads above it, the FFMA EPI_GLOBAL epilogue with
    hpt < 4 at 48 channels and on the FFMA core); a single GlobalGraph head; SemCHGraphConv and SemGraphConv with
    out_features != in_features (partial 64-channel mask tiles); LocalGraph and GraphAttentionBlock at 8, 48 and 160
    channels.  Two heads cannot be built: the reference's own module fails there, and so does the drop-in.
  * Whole models: the strided Optimized1f schedule, the dilated one at T = receptive field (needed-only) and beyond,
    the dense ablation, causal forms, J = 15, 16, 17, 19, 28 and 32, 1 to 5 stages, a 5-wide first filter and 8 to
    1056 channels; the 4096-clip headline on a seeded subset of clips; the fused shrink + MPJPE loss.
  * The bars reject a TF32 forward of the headline model.
  * J = 28 and 32 (the raw 32-joint Human3.6M skeleton and a 28-joint subset): eval-mode input and parameter
    gradients and one training step's gradients at kink-free points (tests/kinkfree.py) against fp64 autograd.

Bars: about 4x the worst value measured over the cases of this file on an H100 80GB HBM3 at a 700 W power limit, per
core ('auto': the F16X3 tensor-core GEMMs where the shapes allow, FFMA elsewhere; 'ffma': FFMA everywhere), as
worst measured max / L2 -> bar max / L2:
  sub-modules, auto: 3.8e-7 / 2.2e-7 -> 1.5e-6 / 9e-7       ffma: 7.4e-7 / 3.8e-7 -> 3e-6 / 1.5e-6
  whole models, auto: 9.0e-7 / 6.6e-7 -> 3.6e-6 / 2.6e-6    ffma: 1.5e-6 / 1.2e-6 -> 6e-6 / 4.8e-6
  fused MPJPE loss, relative: 2.4e-7 -> 1e-6
  the TF32 headline measured 1.0e-3 / 8.8e-4, 290x / 340x the auto model bars.
The J = 28 / 32 gradients are held to the bars of tests/kinkfree.py; measured there, worst per-tensor L2 / max
6.8e-6 / 9.4e-6 (auto) and 9.7e-6 / 1.2e-5 (ffma), y 1.8e-6 of max |y|.
Measured errors go to $GAST_TEST_REPORT_DIR/forward_fp64.txt when that is set, and to record_property.
"""
import collections
import ctypes as C
import functools
import os

import numpy as np
import pytest
import torch

from gast_b200 import engine, synth
from oracle import gast_torch_ref as TR
import fp64ref as R
import kinkfree as K

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')

MAX_BAR = {('module', 'auto'): 1.5e-6, ('module', 'ffma'): 3e-6, ('model', 'auto'): 3.6e-6, ('model', 'ffma'): 6e-6}
L2_BAR = {('module', 'auto'): 9e-7, ('module', 'ffma'): 1.5e-6, ('model', 'auto'): 2.6e-6, ('model', 'ffma'): 4.8e-6}
LOSS_BAR = 1e-6


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield 'ffma' if request.param else 'auto'
    engine.set_gemm_core(0)


def report(record_property, name, core, mx, l2, extra=''):
    record_property('max_rel', mx)
    record_property('l2_rel', l2)
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        with open(os.path.join(REPORT_DIR, 'forward_fp64.txt'), 'a') as f:
            f.write('%s %s: max %.3e l2 %.3e %s\n' % (name, core, mx, l2, extra))


def check(record_property, name, core, y, y64, extra='', what='module'):
    mx, l2 = R.errors(y, y64)
    report(record_property, name, core, mx, l2, extra)
    assert mx <= MAX_BAR[what, core] and l2 <= L2_BAR[what, core], (name, core, mx, l2)


def _handle(module):
    return next(iter(module.__dict__['_gast_handles'].values()))


def launch_kinds(module, run):
    """run() twice; -> (output, Counter of the second call's launch kinds on the module's own handle, its
    tensor-core launch count).  Both calls give the same bits."""
    with torch.no_grad():
        y = run()
        h = _handle(module)
        engine._check(h.lib.gast_set_timing(h.h, 1), 'gast_set_timing')
        try:
            y2 = run()
            ms, kinds = (C.c_float * 1024)(), (C.c_int32 * 1024)()
            n = h.lib.gast_get_timings(h.h, 1024, ms, kinds)
        finally:
            h.lib.gast_set_timing(h.h, 0)
    assert n > 0 and torch.equal(y, y2)
    return y, collections.Counter(engine.LAUNCH_KINDS[kinds[i]] for i in range(n)), int(h.lib.gast_last_tc_launch_count(h.h))


def _x(shape, seed):
    return (0.7 * np.random.RandomState(seed).standard_normal(shape)).astype(np.float32)


def _p64(module):
    return R.f64(module.state_dict())


# ------------------------------------------------------------------------------------------------------------------
# sub-modules
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('J', [17, 19, 24])
@pytest.mark.parametrize('C_,inter', [(32, 32), (96, 32), (48, 16), (32, 8), (128, 32)])
def test_multi_global_graph(J, C_, inter, core, record_property):
    from model.global_attention import MultiGlobalGraph
    heads = C_ // inter
    m = MultiGlobalGraph(torch.eye(J), C_, inter, dropout=0.05)
    synth.randomize_module(m, 40 + heads)
    p = _p64(m)
    x = _x((4, 45, J, C_), J + C_)
    m = m.cuda().eval()
    xd = torch.from_numpy(x).cuda()
    y, kinds, tc = launch_kinds(m, lambda: m(xd))
    with torch.no_grad():
        y64 = TR.multi_global_graph(torch.from_numpy(x).double(), p, '')
    assert kinds['rowdot'] == 1
    if core == 'ffma' or C_ % 32:
        # C = 48: K = 48 is no multiple of the tensor-core K stage, every GEMM runs on FFMA
        assert kinds['gemm_ffma_global'] == 1 and tc == 0, kinds
    elif J <= 20:
        assert kinds['global_mix'] == 1 and kinds['gemm_tc_plain'] == 2 and not kinds['gemm_ffma_global'], kinds
    else:
        assert kinds['gemm_tc_global'] == 1 and not kinds['global_mix'] and not kinds['gemm_ffma_global'], kinds
    check(record_property, 'mglobal_J%d_C%d_h%d' % (J, C_, heads), core, y.cpu(), y64, dict(kinds))


def test_multi_global_graph_two_heads_cannot_be_built():
    """in // inter == 2 makes inter == in // 2, where each head's g conv is in_channels wide (global_attention.py:
    21-24): the reference's concatenation of the heads then does not fit its view, and the drop-in refuses the
    parameter shapes"""
    from model.global_attention import MultiGlobalGraph
    m = MultiGlobalGraph(torch.eye(17), 64, 32, dropout=0.05)
    assert m.num_non_local == 2 and m.attentions[0].g_channels == 64
    with pytest.raises(RuntimeError):
        with torch.no_grad():
            m.cuda().eval()(torch.zeros(2, 3, 17, 64, device='cuda'))


@pytest.mark.parametrize('C_,inter', [(32, 8), (96, 32), (48, 16)])
def test_global_graph_head(C_, inter, core, record_property):
    from model.global_attention import GlobalGraph
    J = 19
    g = GlobalGraph(torch.eye(J), C_, inter)
    synth.randomize_module(g, 50)
    p = _p64(g)
    x = _x((150, C_, J), C_)
    g = g.cuda()
    xd = torch.from_numpy(x).cuda()
    y, kinds, tc = launch_kinds(g, lambda: g(xd))
    with torch.no_grad():
        y64 = TR.global_graph(torch.from_numpy(x).double(), p, '')
    if core == 'ffma' or C_ % 32:
        assert kinds['gemm_ffma_global'] == 1 and tc == 0, kinds
    else:
        assert kinds['gemm_tc_global'] == 1 and tc == 1, kinds
    check(record_property, 'global_C%d_i%d' % (C_, inter), core, y.cpu(), y64, dict(kinds))


@pytest.mark.parametrize('shared', [False, True], ids=['semch', 'semgc'])
@pytest.mark.parametrize('cout', [4, 36, 64, 200])
@pytest.mark.parametrize('cin', [32, 48])
def test_semch_out_width(cin, cout, shared, core, record_property):
    from model.local_attention import SemCHGraphConv, local_adjacencies
    from model.sem_graph_conv import SemGraphConv
    J = 17 if cout in (4, 64) else 19
    con = local_adjacencies(R.adj(J))[1]
    mod = SemGraphConv(cin, cout, con, bias=True) if shared else SemCHGraphConv(cin, cout, con, bias=True)
    synth.randomize_module(mod, 60 + cout)
    p = _p64(mod)
    x = _x((3, 50, J, cin), cin + cout)
    mod = mod.cuda()
    xd = torch.from_numpy(x).cuda()
    y, kinds, tc = launch_kinds(mod, lambda: mod(xd))
    with torch.no_grad():
        y64 = TR.semch(torch.from_numpy(x).double(), p['W'], p['e'], R.masks(J)[1], p['bias'])
    assert y.shape == (3, 50, J, cout)
    if core == 'ffma' or cin % 32:
        assert kinds['gemm_ffma_semch'] == 1 and tc == 0, kinds
    else:
        assert kinds['gemm_tc_semch'] == 1 and tc == 1, kinds
    check(record_property, '%s_J%d_%dto%d' % ('semgc' if shared else 'semch', J, cin, cout), core, y.cpu(), y64,
          dict(kinds))


@pytest.mark.parametrize('J,C_', [(17, 8), (19, 48), (15, 160)])
@pytest.mark.parametrize('kind', ['local', 'block'])
def test_local_graph_and_block(kind, J, C_, core, record_property):
    from model.gast_net import GraphAttentionBlock
    from model.local_attention import LocalGraph
    masks = R.masks(J)
    if kind == 'local':
        mod = LocalGraph(R.adj(J), C_, C_, 0.05)
        x = _x((3, 40, J, C_), C_)
    else:
        mod = GraphAttentionBlock(R.adj(J), C_, C_, 0.05)
        x = _x((3, C_, 40, J), C_)
    synth.randomize_module(mod, 70)
    p = _p64(mod)
    mod = mod.cuda().eval()
    xd = torch.from_numpy(x).cuda()
    y, kinds, tc = launch_kinds(mod, lambda: mod(xd))
    with torch.no_grad():
        x64 = torch.from_numpy(x).double()
        y64 = (TR.local_graph(x64, p, '', masks) if kind == 'local' else TR.graph_attention_block(x64, p, '', masks))
    if core == 'ffma' or C_ == 8:
        assert tc == 0 and kinds['gemm_ffma_semch'] == 1, kinds
    elif C_ == 48:
        # SemCH over K = 48 on FFMA, the 1x1 convolutions over 2C = 96 (and 3C = 144 is not a multiple of 32) split
        assert kinds['gemm_ffma_semch'] == 1 and kinds['gemm_tc_plain'] >= 1, kinds
    else:
        assert tc == sum(kinds.values()) - kinds['rowdot'] - kinds['global_mix'] and kinds['gemm_tc_semch'] == 1, kinds
    check(record_property, '%s_J%d_C%d' % (kind, J, C_), core, y.cpu(), y64, dict(kinds))


# ------------------------------------------------------------------------------------------------------------------
# whole models
# ------------------------------------------------------------------------------------------------------------------
# name: (J, filter widths, channels, B, T, strided, causal, dense)
MODELS = {
    'o1f_j17_c128_T27': (17, [3, 3, 3], 128, 40, 27, True, False, False),
    'dilated_rf_j15_c48_T27': (15, [3, 3, 3], 48, 9, 27, False, False, False),
    'dilated_j19_c160_T60': (19, [3, 3, 3], 160, 2, 60, False, False, False),
    'dense_j16_c48_T30': (16, [3, 3, 3], 48, 3, 30, False, False, True),
    'causal_dilated_j17_c128_T45': (17, [3, 3, 3], 128, 2, 45, False, True, False),
    'causal_o1f_j19_c8_T9': (19, [3, 3], 8, 11, 9, True, True, False),
    'fw3_j17_c128_T3': (17, [3], 128, 50, 3, False, False, False),
    'fw3_dilated_j16_c160_T12': (16, [3], 160, 3, 12, False, False, False),
    'fw33_o1f_j17_c1056_T9': (17, [3, 3], 1056, 3, 9, True, False, False),
    'fw3333_o1f_j16_c64_T81': (16, [3, 3, 3, 3], 64, 5, 81, True, False, False),
    'fw33333_o1f_j17_c32_T243': (17, [3, 3, 3, 3, 3], 32, 2, 243, True, False, False),
    'fw33333_dilated_j15_c8_T250': (15, [3, 3, 3, 3, 3], 8, 1, 250, False, False, False),
    'fw53_dilated_j17_c48_T20': (17, [5, 3], 48, 3, 20, False, False, False),
    'fw53_causal_o1f_j19_c160_T15': (19, [5, 3], 160, 6, 15, True, True, False),
    'o1f_j28_c128_T27': (28, [3, 3, 3], 128, 12, 27, True, False, False),
    'dilated_j32_c48_T20': (32, [3, 3], 48, 3, 20, False, False, False),
}


def build_model(J, fw, ch, strided, causal, dense, seed=7):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    if strided:
        m = SpatioTemporalModelOptimized1f(R.adj(J), J, 2, J, fw, causal=causal, dropout=0.05, channels=ch)
    else:
        m = SpatioTemporalModel(R.adj(J), J, 2, J, fw, causal=causal, dropout=0.05, channels=ch, dense=dense)
    synth.randomize_module(m, seed)
    return m.eval()


@functools.lru_cache(maxsize=None)
def model_reference(name):
    """(state_dict, x, fp64 output) of MODELS[name]"""
    J, fw, ch, B, T, strided, causal, dense = MODELS[name]
    with pytest.MonkeyPatch.context() as mp:
        R.install_tables(mp, J)
        sd = build_model(J, fw, ch, strided, causal, dense).state_dict()
    x = synth.synth_input(B, T, J, 2, seed=100 + J)
    return sd, x, R.model_forward64(sd, x, J, fw, causal, strided, dense)


@pytest.mark.parametrize('name', sorted(MODELS))
def test_model_forward(name, core, record_property, monkeypatch):
    J, fw, ch, B, T, strided, causal, dense = MODELS[name]
    sd, x, y64 = model_reference(name)
    R.install_tables(monkeypatch, J)
    m = build_model(J, fw, ch, strided, causal, dense)
    m.load_state_dict(sd)
    m = m.cuda()
    xd = torch.from_numpy(x).cuda()
    y, kinds, tc = launch_kinds(m, lambda: m(xd))
    assert y.shape == y64.shape
    if core == 'ffma':
        assert tc == 0
    elif ch % 32 == 0:
        assert tc > 0 and kinds['gemm_tc_semch'] == len(fw), kinds
    check(record_property, name, core, y.cpu(), y64, 'tc %d' % tc, what='model')


HEADLINE = (17, [3, 3, 3], 128, False, False, False)    # bench.py: SpatioTemporalModel, 27 frames, 4096 clips
HEADLINE_B = 4096


def headline_subset():
    """a seeded set of 64 of the 4096 clips: the first two, the last and 61 others.  A clip's 9 expand frames are
    153 rows, so each one straddles a 128-row tile of the flat GEMMs and a 7-frame (119-row) tile of the
    frame-structured ones; the 4096 clips take several waves of either."""
    rs = np.random.RandomState(5)
    pick = {0, 1, HEADLINE_B - 1} | set((2 + rs.choice(HEADLINE_B - 3, 61, replace=False)).tolist())
    return sorted(pick)


@functools.lru_cache(maxsize=None)
def headline_reference():
    J, fw, ch, strided, causal, dense = HEADLINE
    sd = build_model(*HEADLINE, seed=1).state_dict()
    x = synth.synth_input(HEADLINE_B, 27, J, 2, seed=1234)
    idx = headline_subset()
    return sd, x, idx, R.model_forward64(sd, x[idx], J, fw)


def test_headline_batch_subset(core, record_property):
    sd, x, idx, y64 = headline_reference()
    assert len(idx) == 64
    m = build_model(*HEADLINE, seed=1)
    m.load_state_dict(sd)
    m = m.cuda()
    xd = torch.from_numpy(x).cuda()
    y, kinds, tc = launch_kinds(m, lambda: m(xd))
    assert y.shape == (HEADLINE_B, 1, 17, 3)
    assert (tc > 0) == (core == 'auto')
    check(record_property, 'headline_4096_subset64', core, y[idx].cpu(), y64, 'tc %d' % tc, what='model')
    # the fused shrink + MPJPE (run_model_mpjpe): over the whole batch against the fp64 MPJPE of the same call's poses,
    # and against the fp64 model's MPJPE on the subset
    tgt = torch.from_numpy(synth.synth_target(HEADLINE_B, 17, seed=9)).cuda()
    with torch.no_grad():
        yl, loss = engine.run_model_mpjpe(m, xd, tgt)
        assert torch.equal(yl, y)
        ysub, lsub = engine.run_model_mpjpe(m, xd[idx].contiguous(), tgt[idx].contiguous())
    t64 = tgt.cpu().double()
    l_own = float(torch.norm(yl.cpu().double() - t64, dim=3).mean())
    l_64 = float(torch.norm(y64 - t64[idx], dim=3).mean())
    e_own, e_64 = abs(float(loss) - l_own) / l_own, abs(float(lsub) - l_64) / l_64
    record_property('loss_rel_own', e_own)
    record_property('loss_rel_fp64', e_64)
    report(record_property, 'headline_loss', core, e_own, e_64, '(relative loss errors: own poses, fp64 subset)')
    assert e_own <= LOSS_BAR and e_64 <= LOSS_BAR, (e_own, e_64)


def test_tf32_headline_fails_the_fp32_bar(record_property):
    """the bars discriminate: one TF32 product per multiply-add (about 1e-3 off) is rejected by them"""
    sd, x, idx, y64 = headline_reference()
    m = build_model(*HEADLINE, seed=1)
    m.load_state_dict(sd)
    m = engine.set_precision(m.cuda(), 'tf32')
    with torch.no_grad():
        y = m(torch.from_numpy(x[idx]).cuda()).cpu()
    mx, l2 = R.errors(y, y64)
    report(record_property, 'headline_tf32', 'auto', mx, l2)
    assert mx > 10 * MAX_BAR['model', 'auto'] and l2 > 10 * L2_BAR['model', 'auto'], (mx, l2)


# ------------------------------------------------------------------------------------------------------------------
# J = 28 and 32: the backward's attention adjoint (att_mix_bwd_kernel) takes 16 J^2 floats of shared memory
# ------------------------------------------------------------------------------------------------------------------
MANY_JOINTS = {
    'j28_dilated_eval': K.Case(28, [3, 3, 3], 32, 2, 27, False, False, False, False),
    'j32_o1f_eval': K.Case(32, [3, 3], 32, 3, 9, True, False, False, False),
    'j28_o1f_train': K.Case(28, [3, 3], 32, 4, 9, True, False, False, True),
    'j32_o1f_train': K.Case(32, [3, 3, 3], 32, 3, 27, True, False, False, True),
}


def _many_joint_module(case):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    kls = SpatioTemporalModelOptimized1f if case.strided else SpatioTemporalModel
    m = kls(R.adj(case.J), case.J, 2, case.J, case.fw, causal=case.causal, dropout=0.0, channels=case.ch)
    synth.randomize_module(m, 5)
    return m.train(case.training)


@pytest.mark.parametrize('name', sorted(MANY_JOINTS))
def test_many_joint_gradients(name, core, record_property, monkeypatch):
    case = MANY_JOINTS[name]
    R.install_tables(monkeypatch, case.J)
    monkeypatch.setattr(K, 'masks', R.masks)
    m = _many_joint_module(case)
    x = K.inputs(case)
    sd, (relu, leaky, _) = K.make_kink_free(m.state_dict(), x, case)
    assert relu >= K.MARGIN and leaky >= K.MARGIN, (relu, leaky)
    with torch.no_grad():
        shape = K.port_forward(R.f64(sd), x.double(), case).shape
    tgt = K.target(shape)
    y64, loss64, g64, scales = K.port_grads(sd, x, tgt, case, torch.float64)
    m.load_state_dict(sd)
    m = m.cuda().train(case.training)
    xd = x.cuda().requires_grad_()
    y = m(xd)
    loss = torch.mean(torch.norm(y - tgt.cuda(), dim=3))
    loss.backward()
    torch.cuda.synchronize()
    got = {k: p.grad.cpu().double() for k, p in m.named_parameters()}
    got['x'] = xd.grad.cpu().double()
    mx, l2 = R.errors(y.detach().cpu(), y64)
    bad, err = K.check(got, g64, scales, core if core == 'ffma' else 'tc')
    worst = max(v[0] for v in err.values() if v[0] is not None), max(v[1] for v in err.values() if v[0] is not None)
    report(record_property, name, core, mx, l2, 'grad worst l2 %.2e max %.2e' % worst)
    assert mx <= K.Y_BAR, mx
    assert abs(loss.item() - loss64) / abs(loss64) <= K.LOSS_BAR
    assert not bad, sorted(bad, key=lambda t: -(t[1] or 0))[:12]
