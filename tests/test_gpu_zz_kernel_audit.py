"""GPU: every expand, theta/phi row-dot, attention-mix and shrink launch of the forward, mpjpe, chunked, training and
stream calls, each held to fp64 of its own operands (tests/kernelaudit.py), in fp32, TF32, at the fp16 precision
(set_precision('fp16')) and in half models (model.half()).

gast_debug_set_kernel_audit is set on every library handle the engine creates while this file runs; each launch is
snapshotted before it runs and checked element by element after it, at the bound of its arithmetic, and for the
columns of its output window it does not own.  A failure names the launch and the element.  Calls:
  * batched forwards in all four forms: a first filter width of 5 (expand_rows_kernel<10>) at 96 channels (256 % 24
    != 0: surplus expand threads), 1056 channels (two expand chunks, a 2112-wide block: rowdot_kernel<8>, and a mix of
    one frame per CTA), J = 15, 16, 19 and 20 (the mix at MIX_JMAX: every padded slot of an attention row), row counts
    that are not multiples of 128 and frame counts that are not multiples of the mix's frames per CTA;
  * MultiGlobalGraph with 1 and 3 heads (rowdot_kernel<2/6>) and a GlobalGraph head, fp32.  Two heads need
    inter = in / 2, where GlobalGraph widens g to all in channels (model/global_attention.py) and the library refuses
    the module at gast_prepare, so no call reaches rowdot_kernel<4>;
  * run_model_mpjpe at 15 rows (two blocks: a single block needs at most 8 rows, which no model of 15 or more joints
    makes) and at 10,200 rows (the grid capped at 1024 blocks, each striding), each called twice for the same loss
    bit for bit (the ticket reset);
  * run_model_chunked with a window that does not divide T_out;
  * streams at fp32 and fp16: single pushes (expand over one window: T = k0, T0 = 1), push_frames (T0 = K windows),
    peek, a subset push, and the graphed pool (the device-table push) whose eager tick is audited and whose captured
    ticks are skipped;
  * the training forward's row dots (fp32);
  * the ends of fp16's range: a half model whose input is scaled so that the expand outputs reach fp16's top binade
    and inf, and then its subnormals (only the expand is audited there).
Outputs with the audit on are bitwise those with it off.  We / be and U / cab are held to fp64 of the module
parameters (kernelaudit.fold_bounds, collapse_bounds).  The last test asserts that the audited launches reached every
tag in COVERAGE and writes the worst err / bound per kind and form to $GAST_TEST_REPORT_DIR/kernel_audit.txt.

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit: 682 launches audited and 12 captured ones skipped in
about 30 s; worst err / bound per kind in fp32 / TF32 / fp16 precision / half:
  expand 0.44 / 0.37 / 0.996 / 0.994;  rowdot 0.32 / 0.20 / 0.25 / 0.18;  mix 0.19 / 0.15 / 0.994 / 0.990
  shrink 0.10 / 0.11 / 0.12 / 0.97;  shrink_mpjpe y 0.15 (fp32) / 0.15 (fp16), loss 0.11 / 0.13
An fp16 output's bound is the fp32 bound plus half an fp16 ulp, and the rounding to fp16 takes nearly all of that
half ulp for some element of every large launch, so the fp16 margins sit just under 1 by construction.
"""
import collections
import subprocess
import weakref

import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth
import kernelaudit as KA

pytestmark = pytest.mark.gpu

STATE = {'records': [], 'skips': 0, 'cases': set(), 'derived': collections.Counter()}
CASE_NAMES = {'models', 'edges', 'modules', 'mpjpe', 'chunked', 'streams', 'graphed', 'train', 'range'}
FORMS = ('fp32', 'tf32', 'fp16', 'half')

COVERAGE = [
    'expand:kft6:f32->f32', 'expand:kft10:f32->f32', 'expand:kft6:f32->f16', 'expand:kft10:f32->f16',
    'expand:kft6:f16->f16', 'expand:kft10:f16->f16',
    'rowdot:rowdot8:f32->f32', 'rowdot:rowdot8:f16->f32', 'rowdot:rowdot<8>:f32->f32', 'rowdot:rowdot<8>:f16->f32',
    'rowdot:rowdot<2>:f32->f32', 'rowdot:rowdot<6>:f32->f32',
    'mix:mix:f32->f32', 'mix:mix:f16->f16',
    'shrink:shrink:f32->f32', 'shrink:shrink:f16->f32', 'shrink:shrink:f16->f16',
    'shrink_mpjpe:shrink_mpjpe:f32->f32', 'shrink_mpjpe:shrink_mpjpe:f16->f32',
    'expand:two_chunks:f32', 'expand:two_chunks:f16', 'expand:surplus_threads', 'expand:partial_block',
    'expand:one_window', 'expand:stride1_windows',
    'mix:J15', 'mix:J16', 'mix:J17', 'mix:J19', 'mix:J20', 'mix:fpb1', 'mix:partial_block',
    'shrink_mpjpe:blocks', 'shrink_mpjpe:grid_stride',
    'range:inf', 'range:top_binade', 'range:subnormal',
]

HANDLES = weakref.WeakSet()     # every library handle the engine creates while this file runs


@pytest.fixture(autouse=True, scope='module')
def _register_handles():
    orig = engine._Handle.__init__

    def init(h, *a, **k):
        orig(h, *a, **k)
        HANDLES.add(h)
    engine._Handle.__init__ = init
    yield
    engine._Handle.__init__ = orig


class _Audit(object):
    """the auditor on every live handle, and on each handle created while it is active"""

    def __init__(self, **kw):
        self.aud = KA.Auditor(**kw)
        self._orig = engine._Handle.__init__

    def __enter__(self):
        orig, me = self._orig, self

        def init(h, *a, **k):
            orig(h, *a, **k)
            me.aud.install(h.lib, h.h)
        engine._Handle.__init__ = init
        self.skips0 = self._skips()
        self.on()
        return self

    def _skips(self):
        return sum(int(h.lib.gast_debug_kernel_audit_skips(h.h)) for h in list(HANDLES))

    def __exit__(self, *exc):
        engine._Handle.__init__ = self._orig
        STATE['skips'] += self._skips() - self.skips0
        self.off()

    def off(self):
        for h in list(HANDLES):
            h.lib.gast_debug_set_kernel_audit(h.h, _lib.KernelAuditFn(), None)

    def on(self):
        for h in list(HANDLES):
            self.aud.install(h.lib, h.h)


def _same(a, b):
    if isinstance(a, (tuple, list)):
        return all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, torch.Tensor):
        return torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.isnan(), b.isnan())
    return True


def audited(run, form='fp32', exact=True, **kw):
    """run() with the audit on, then again with it off: the same bits.  -> the audit (records, kept launches)"""
    with _Audit(**kw) as A:
        try:
            y1 = run()
        except engine.GastError as ex:
            raise AssertionError('%s\n%s' % (ex, A.aud.failure)) from ex
        torch.cuda.synchronize()
        assert A.aud.failure is None, A.aud.failure
        assert A.aud.records, 'no kernel launch was audited'
        A.off()
        y2 = run()
        torch.cuda.synchronize()
    assert not exact or _same(y1, y2), 'outputs with the audit on differ from those with it off'
    for r in A.aud.records:
        r['form'] = form
    STATE['records'] += A.aud.records
    return A.aud


def _build(J, fw, ch, strided=False, causal=False, seed=7):
    from test_gpu_forward_fp64 import build_model
    if J != 20:
        return build_model(J, fw, ch, strided, causal, False, seed=seed)
    # 20 joints, the most the mix kernel takes: the 19-joint skeleton with one more leaf on the root (no model of the
    # reference has 20 joints; LocalGraph needs a joint table for it, see _table20)
    from common.graph_utils import adj_mx_from_skeleton
    from common.skeleton import Skeleton
    from model.gast_net import SpatioTemporalModel
    adj = adj_mx_from_skeleton(Skeleton(PARENTS20, [], []))
    m = SpatioTemporalModel(adj, 20, 2, 20, fw, causal=causal, dropout=0.05, channels=ch)
    synth.randomize_module(m, seed)
    return m.eval()


PARENTS20 = list(synth.skeleton_parents(19)) + [0]


def _tables(monkeypatch, J):
    """the joint table LocalGraph needs for J (fp64ref's for 28 / 32; for 20 the leaves are the distal joints)"""
    import fp64ref as R
    import model.local_attention as LA
    if J == 20 and J not in LA._JOINT_TABLES:
        monkeypatch.setitem(LA._JOINT_TABLES, 20, ([j for j in range(20) if j not in PARENTS20], [], []))
    elif J != 20:
        R.install_tables(monkeypatch, J)


def _in_form(m, x, form):
    """(model, input) on the GPU in `form`"""
    m = m.cuda()
    if form == 'half':
        return m.half(), x.half()
    return engine.set_precision(m, form), x


def _forward(m, x):
    with torch.no_grad():
        return m(x).clone()


def _derived(aud, sd, prefix=''):
    """hold the We / be and U / cab that the kept launches read to fp64 of the state dict (numpy)"""
    for P, S, _ in aud.launches:
        if KA.KINDS[P['kind']] == 'expand' and 'expand_conv.weight' in sd:
            We64, eWe, be64, ebe = KA.fold_bounds(sd, P['taps'], P['Fin'])
            KA.within(S['We'], We64, eWe, 'We')
            KA.within(S['be'], be64, ebe, 'be')
            STATE['derived']['fold'] += 1
        if KA.KINDS[P['kind']] == 'rowdot':
            gp = prefix if 'expand_conv.weight' not in sd else \
                'layers_graph_conv.%d.global_graph_layer.' % P['block']
            for h in range(P['heads']):
                hp = gp if P['heads'] == 1 and gp + 'theta.weight' in sd else gp + 'attentions.%d.' % h
                U64, eU, cab64, ecab = KA.collapse_bounds(sd[hp + 'theta.weight'], sd[hp + 'theta.bias'],
                                                          sd[hp + 'phi.weight'], sd[hp + 'phi.bias'],
                                                          sd[hp + 'concat_project.0.weight'].ravel())
                KA.within(S['U'][2 * h:2 * h + 2], U64, eU, 'U of head %d' % h)
                KA.within(S['cab'][2 * h:2 * h + 2], cab64, ecab, 'cab of head %d' % h)
            STATE['derived']['collapse'] += 1


def _sd(m):
    return {k: v.detach().float().cpu().numpy() for k, v in m.state_dict().items()}


# ------------------------------------------------------------------------------------------------------------------
# batched forwards
# ------------------------------------------------------------------------------------------------------------------
# (J, filter widths, channels, B, T, strided, causal)
MODELS = {
    'fw53_j17_c96': (17, [5, 3], 96, 3, 17, False, False),
    'j15_c64_causal': (15, [3, 3], 64, 2, 13, False, True),
    'j16_c32_o1f': (16, [3, 3], 32, 5, 9, True, False),
    'j19_c64': (19, [3, 3], 64, 1, 12, False, False),
    'j20_c32': (20, [3, 3], 32, 2, 11, False, False),     # _build: a 20-joint skeleton
}


@pytest.mark.parametrize('form', FORMS)
def test_model_forwards(form, monkeypatch):
    for name, (J, fw, ch, B, T, strided, causal) in sorted(MODELS.items()):
        _tables(monkeypatch, J)
        m0 = _build(J, fw, ch, strided, causal)
        sd = _sd(m0)
        m, x = _in_form(m0, torch.from_numpy(synth.synth_input(B, T, J, 2, seed=100 + J)).cuda(), form)
        aud = audited(lambda: _forward(m, x), form, keep=form == 'fp32')
        if form == 'fp32':
            _derived(aud, sd)
    STATE['cases'].add('models')


@pytest.mark.parametrize('form', FORMS)
def test_wide_model(form):
    """1056 channels: two expand chunks, a 2112-wide second block (rowdot_kernel<8>) and one frame per mix CTA"""
    m, x = _in_form(_build(17, [3, 3], 1056, True), torch.from_numpy(synth.synth_input(1, 9, 17, 2, seed=4)).cuda(),
                    form)
    aud = audited(lambda: _forward(m, x), form)
    assert any(r['kind'] == 'rowdot' and r['variant'] == 8 for r in aud.records)
    STATE['cases'].add('edges')


def test_sub_modules():
    from model.global_attention import GlobalGraph, MultiGlobalGraph
    for J, C_, inter in ((17, 32, 32), (19, 96, 32)):     # 1 and 3 heads
        m = MultiGlobalGraph(torch.eye(J), C_, inter, dropout=0.05)
        synth.randomize_module(m, 40 + J)
        sd = _sd(m)
        m = m.cuda().eval()
        x = torch.from_numpy((0.7 * np.random.RandomState(J).standard_normal((3, 7, J, C_))).astype(np.float32)).cuda()
        _derived(audited(lambda: _forward(m, x), keep=True), sd)
    g = GlobalGraph(torch.eye(19), 96, 32)
    synth.randomize_module(g, 50)
    sd = _sd(g)
    g = g.cuda()
    xg = torch.from_numpy((0.7 * np.random.RandomState(5).standard_normal((30, 96, 19))).astype(np.float32)).cuda()
    _derived(audited(lambda: _forward(g, xg), keep=True), sd)
    STATE['cases'].add('modules')


# ------------------------------------------------------------------------------------------------------------------
# mpjpe, chunked, training
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('form', ['fp32', 'fp16'])
def test_mpjpe(form, monkeypatch):
    for J, B, T in ((15, 1, 9), (17, 600, 9)):
        _tables(monkeypatch, J)
        m, x = _in_form(_build(J, [3, 3], 32, True), torch.from_numpy(synth.synth_input(B, T, J, 2, seed=J)).cuda(),
                        form)
        tgt = torch.from_numpy(np.random.RandomState(J).standard_normal((B, 1, J, 3)).astype(np.float32)).cuda()

        def run():
            with torch.no_grad():
                y, l1 = engine.run_model_mpjpe(m, x, tgt)
                l1 = l1.clone()
                _, l2 = engine.run_model_mpjpe(m, x, tgt)
            assert torch.equal(l1.view(torch.int32), l2.view(torch.int32)), (float(l1), float(l2))
            return [y.clone(), l1]
        aud = audited(run, form)
        assert any(r['loss_worst'] is not None for r in aud.records)
    STATE['cases'].add('mpjpe')


@pytest.mark.parametrize('form', FORMS)
def test_chunked(form):
    m, x = _in_form(_build(17, [3, 3], 64, False), torch.from_numpy(synth.synth_input(2, 20, 17, 2, seed=8)).cuda(),
                    form)
    with torch.no_grad():
        audited(lambda: engine.run_model_chunked(m, x, 5).clone(), form)        # T_out = 12
    STATE['cases'].add('chunked')


def test_training_rowdot():
    import kinkfree as K
    case = K.CASES['o1f_j17_c128_train']              # strided: the step repeats bit for bit
    m = K.module(case).cuda()
    x = torch.as_tensor(K.inputs(case)).float().cuda()
    sd = {k: v.clone() for k, v in m.state_dict().items()}

    def run():
        m.load_state_dict(sd)
        m.zero_grad(set_to_none=True)
        y = m(x)
        (y * y).sum().backward()
        return [y.detach().clone()] + [p.grad.clone() for p in m.parameters() if p.grad is not None]
    aud = audited(run)
    assert {r['kind'] for r in aud.records} == {'rowdot'}
    STATE['cases'].add('train')


# ------------------------------------------------------------------------------------------------------------------
# streams
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('form', ['fp32', 'fp16'])
def test_streams(form):
    from gast_b200.realtime import CausalStream, PoseStream
    for J, causal in ((17, True), (19, False)):
        m = engine.set_precision(_build(J, [3, 3], 64, False, causal).cuda(), form)
        n = 3
        frames = torch.from_numpy(synth.synth_input(n, 20, J, 2, seed=J)).cuda()

        def run():
            ps = CausalStream(m, n) if causal else PoseStream(m, n)
            out = []
            with torch.no_grad():
                for t in range(11):                       # the 9-frame ring wraps
                    out.append(ps.push(frames[:, t]))
                out.append(ps.push_frames(frames[:, 11:16].contiguous()))
                if not causal:
                    out.append(ps.peek(2))
                out.append(ps.push(frames[[0, 2], 16], streams=[0, 2]))
            return [o[0] if isinstance(o, tuple) else o for o in out]
        audited(run, form)
    STATE['cases'].add('streams')


@pytest.mark.parametrize('form', ['fp32', 'fp16'])
def test_graphed_pool(form):
    from gast_b200.realtime import GraphedPoseStream
    m = engine.set_precision(_build(19, [3, 3], 32, False, False).cuda(), form)
    frames = torch.from_numpy(synth.synth_input(2, 12, 19, 2, seed=3)).cuda()
    skips0 = STATE['skips']

    def run():
        gs = GraphedPoseStream(m, 2, K=2)
        with torch.no_grad():
            return [gs.push(frames[:, 2 * t:2 * t + 2].contiguous())[0] for t in range(5)]
    audited(run, form)
    assert STATE['skips'] > skips0, 'no launch ran under capture'
    STATE['cases'].add('graphed')


# ------------------------------------------------------------------------------------------------------------------
# the ends of fp16's range
# ------------------------------------------------------------------------------------------------------------------
def test_fp16_range_ends():
    """a half model with be = 0 (the input and expand BatchNorms shift nothing), so that the expand outputs scale with
    the input: scaled to reach 2^17 they fill fp16's top binade and overflow to inf, scaled to 2^-16 they are
    subnormal; round to nearest decides each element against 65520"""
    m = _build(17, [3, 3], 32, True)
    with torch.no_grad():
        for bn in (m.init_bn, m.expand_bn):
            bn.bias.zero_()
            bn.running_mean.zero_()
    sd = _sd(m)
    We64 = KA.fold_bounds(sd, 3, 2)[0]
    x0 = synth.synth_input(2, 9, 17, 2, seed=12).astype(np.float64)
    # the strided expand's windows: frames 3 t0 .. 3 t0 + 2, one row (kk, i) per output position (b, t0, j)
    taps = x0.reshape(2, 3, 3, 17, 2).transpose(0, 1, 3, 2, 4).reshape(-1, 6)
    peak = float(np.abs(taps @ We64).max())
    assert np.abs(x0).max() * 2.0 ** 17 / peak < 65504, 'the scaled input must stay finite in fp16'
    m = m.cuda().half()
    for scale, tag in ((2.0 ** 17 / peak, 'top'), (2.0 ** -16 / peak, 'sub')):
        x = torch.from_numpy(x0 * scale).half().cuda()
        aud = audited(lambda: _forward(m, x), 'half', kinds=('expand',), keep=True)
        (P, S, out1), = aud.launches
        y = out1[:, :P['K']]
        if tag == 'top':
            assert np.isinf(y).any() and ((y >= 32768) & np.isfinite(y)).any()
            STATE['records'][-1]['tags'] |= {'range:inf', 'range:top_binade'}
        else:
            assert ((y > 0) & (y < 2.0 ** -14)).any()
            STATE['records'][-1]['tags'] |= {'range:subnormal'}
    STATE['cases'].add('range')


# ------------------------------------------------------------------------------------------------------------------
# coverage and the record
# ------------------------------------------------------------------------------------------------------------------
def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = 'unknown'
    return '%s, power limit %s' % (name, pl or 'unknown')


def test_zz_coverage_and_report():
    if STATE['cases'] != CASE_NAMES:
        pytest.skip('coverage needs every call of this file (ran: %s)' % sorted(STATE['cases']))
    recs = STATE['records']
    seen = collections.Counter()
    worst = collections.defaultdict(lambda: [0.0, 0.0, 0])
    for r in recs:
        for t in r['tags']:
            seen[t] += 1
        w = worst[(r['kind'], r['form'])]
        w[0] = max(w[0], r['worst'])
        w[1] = max(w[1], r['loss_worst'] or 0.0)
        w[2] += 1
    lines = ['# %s: %d launches audited, %d skipped under capture; derived constants checked: %s\n' % (
        _card(), len(recs), STATE['skips'], dict(STATE['derived']))]
    lines += ['# %-40s %d\n' % (k, v) for k, v in sorted(seen.items())]
    lines += ['# worst %-12s %-4s: err/bound %.3e (loss %.3e) over %d\n' % (k + tuple(v)) for k, v in
              sorted(worst.items())]
    _write_report(lines + [KA.report_line(r) for r in recs])
    print(''.join(lines))
    missing = [k for k in COVERAGE if not seen[k]]
    assert not missing, 'tags no audited launch reached: %s' % missing
    assert STATE['derived']['fold'] and STATE['derived']['collapse']


def _write_report(lines):
    import gemmaudit as GA
    GA.write_report(lines, 'kernel_audit.txt')
