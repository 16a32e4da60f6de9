"""GPU: every GEMM launch of the forward, training, gradient, chunked and stream calls, each held to fp64 of its own
fp32 operands (tests/gemmaudit.py), on both GEMM cores.

gast_debug_set_gemm_audit is set on every library handle the engine creates while this file runs; each launch_gemm
launch is snapshotted before it runs and checked element by element after it, at the bound of the core and form that
ran, against the emulation of its tensor-core form, and for the columns of its output window it does not own.  A
failure names the launch and the element.  Calls:
  * the batched forward of the sixteen model geometries of test_gpu_forward_fp64.py and of the headline model at
    256 clips, MultiGlobalGraph with 1, 3 and 4 heads at J = 17, 19 and 24, a GlobalGraph head, SemCHGraphConv with
    Cout != Cin; fp32-grade and TF32;
  * training forward and backward at kinkfree.CASES geometries, fp32-grade (3xTF32 on the training copies) and TF32;
  * the eval backward, and the chunked forward and backward with a window that does not divide T_out;
  * streams: push, push_frames, peek and a subset push of a causal and a non-causal stream (a ring that wraps, J = 17
    and 19), and the graphed pool, whose eager warm-up tick is audited and whose captured ticks are counted as skipped.
Each call runs on the tensor-core core (gemm core 0) and on FFMA (core 1); its outputs with the audit on are bitwise
those with it off.  The last test asserts that the audited launches reached every form listed in COVERAGE.

Forms of the GemmP contract that no real call makes, so that only tests/test_gemmaudit_cpu.py's host launches carry
them: two A segments (the only concatenation, the block's cat conv, has three), and with it a plain launch that mixes
TMA-fed and gathered segments; an A segment frame map with t_off != 0 (the offsets are the residual maps'); an output
whose ld_out exceeds the columns the launch owns (every output and scratch buffer is dense).

Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, 5,300 launches audited, the captured ticks of the graphed
pool skipped; worst err / bound and relative L2 from fp64 per core and form:
  FFMA plain / SemCH / global: 0.31 / 0.32 / 0.09, L2 9.5e-7 / 6.2e-7 / 2.4e-7
  F16X3 plain / SemCH / global: 0.031 / 0.038 / 0.020, L2 3.6e-7 / 2.0e-7 / 1.4e-7;  3xTF32 plain: 0.064, L2 2.4e-7
  1xTF32 plain / SemCH / global: 0.82 / 0.56 / 0.12, L2 4.9e-4 / 3.1e-4 / 2.0e-4
The 1xTF32 bound is the worst case of one rounding per operand, 2^-10 of |a w|; a short dot product whose largest
term rounds both operands the same way nearly reaches it, so it has no more margin to give.  The full record, with
the card's name and power limit, goes to $GAST_TEST_REPORT_DIR/gemm_audit.txt.
"""
import collections
import subprocess
import weakref

import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth
import gemmaudit as GA

pytestmark = pytest.mark.gpu

STATE = {'records': [], 'skips': 0, 'cases': set()}
CASE_NAMES = {'models', 'headline', 'modules', 'train', 'eval_chunked', 'streams', 'graphed'}

COVERAGE = [
    ('tc', 'plain'), ('tc', 'semch'), ('tc', 'global'), ('ffma', 'plain'), ('ffma', 'semch'), ('ffma', 'global'),
    'form:f16x3', 'form:3xtf32', 'form:tf32',
    'feed_tma', 'feed_gather',
    'nseg3', 'flat', 'frame_tiled',
    'partial_row_tile', 'partial_col_tile', 'N_lt_32',
    'bias', 'relu', 'res_map',
    'tap_stride_t_mul', 'FJ_lt_128',
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

    def __init__(self):
        self.aud = GA.Auditor()
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
        return sum(int(h.lib.gast_debug_gemm_audit_skips(h.h)) for h in list(HANDLES))

    def __exit__(self, *exc):
        engine._Handle.__init__ = self._orig
        STATE['skips'] += self._skips() - self.skips0
        self.off()
        STATE['records'] += self.aud.records

    def off(self):
        for h in list(HANDLES):
            h.lib.gast_debug_set_gemm_audit(h.h, _lib.GemmAuditFn(), None)

    def on(self):
        for h in list(HANDLES):
            self.aud.install(h.lib, h.h)

    def ok(self):
        assert self.aud.failure is None, self.aud.failure


def _same(a, b):
    if isinstance(a, (tuple, list)):
        return all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b) or (a.isnan().any() and torch.equal(a.nan_to_num(), b.nan_to_num()))
    return True


def audited(run, cores=(0, 1), exact=True):
    """run() with the audit on, per core; then again with it off: the same bits (exact=False: a call whose results
    do not repeat bit for bit from run to run even without the audit is not compared)"""
    n0 = len(STATE['records'])
    for core in cores:
        engine.set_gemm_core(core)
        try:
            with _Audit() as A:
                try:
                    y1 = run()
                except engine.GastError as ex:
                    raise AssertionError('%s\n%s' % (ex, A.aud.failure)) from ex
                torch.cuda.synchronize()
                A.ok()
                assert A.aud.records, 'no GEMM launch was audited'
                A.off()
                y2 = run()
                torch.cuda.synchronize()
                A.on()
            assert not exact or _same(y1, y2), 'outputs with the audit on differ from those with it off (core %d)' % core
        finally:
            engine.set_gemm_core(0)
    return STATE['records'][n0:]


def _adj(J):
    import fp64ref as R
    return R.adj(J)


# ------------------------------------------------------------------------------------------------------------------
# batched forward
# ------------------------------------------------------------------------------------------------------------------
def _forward(m, x):
    with torch.no_grad():
        return m(x).clone()


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
def test_model_forwards(prec, monkeypatch):
    import fp64ref as R
    from test_gpu_forward_fp64 import MODELS, build_model
    for name, (J, fw, ch, B, T, strided, causal, dense) in sorted(MODELS.items()):
        R.install_tables(monkeypatch, J)
        m = engine.set_precision(build_model(J, fw, ch, strided, causal, dense).cuda(), prec)
        x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=100 + J)).cuda()
        recs = audited(lambda: _forward(m, x))
        assert recs, name
    STATE['cases'].add('models')


def test_headline_forward():
    from test_gpu_forward_fp64 import HEADLINE, build_model
    m = build_model(*HEADLINE, seed=1).cuda()
    x = torch.from_numpy(synth.synth_input(256, 27, 17, 2, seed=1234)).cuda()
    audited(lambda: _forward(m, x))
    engine.set_precision(m, 'tf32')
    audited(lambda: _forward(m, x), cores=(0,))
    STATE['cases'].add('headline')


def test_sub_modules():
    from model.global_attention import GlobalGraph, MultiGlobalGraph
    from model.local_attention import SemCHGraphConv, local_adjacencies
    for J, C_, inter in ((17, 32, 32), (19, 96, 32), (24, 128, 32)):
        m = MultiGlobalGraph(torch.eye(J), C_, inter, dropout=0.05)
        synth.randomize_module(m, 40 + J)
        m = m.cuda().eval()
        x = torch.from_numpy((0.7 * np.random.RandomState(J).standard_normal((4, 45, J, C_))).astype(np.float32)).cuda()
        audited(lambda: _forward(m, x))
    g = GlobalGraph(torch.eye(19), 96, 32)
    synth.randomize_module(g, 50)
    g = g.cuda()
    xg = torch.from_numpy((0.7 * np.random.RandomState(5).standard_normal((150, 96, 19))).astype(np.float32)).cuda()
    audited(lambda: _forward(g, xg))
    for J, cin, cout in ((17, 32, 36), (19, 64, 200)):
        con = local_adjacencies(_adj(J))[1]
        s = SemCHGraphConv(cin, cout, con, bias=True)
        synth.randomize_module(s, 60 + cout)
        s = s.cuda()
        xs = torch.from_numpy((0.7 * np.random.RandomState(cout).standard_normal((3, 50, J, cin))).astype(
            np.float32)).cuda()
        audited(lambda: _forward(s, xs))
    STATE['cases'].add('modules')


# ------------------------------------------------------------------------------------------------------------------
# training and gradients
# ------------------------------------------------------------------------------------------------------------------
TRAIN_CASES = ['o1f_j17_c128_train', 'o1f_j19_c160_train', 'dilated_rf_j16_c128_train', 'causal_T40_j17_c48_train',
               'o1f_j16_c16_train']


@pytest.mark.parametrize('tprec', ['fp32', 'tf32'])
def test_training(tprec):
    import kinkfree as K
    for name in TRAIN_CASES:
        case = K.CASES[name]
        m = engine.set_training_precision(K.module(case).cuda(), tprec)
        x = torch.as_tensor(K.inputs(case)).float().cuda()

        def step():
            m.zero_grad(set_to_none=True)
            y = m(x)
            (y * y).sum().backward()
            return [y.detach().clone()] + [p.grad.clone() for p in m.parameters() if p.grad is not None]
        sd = {k: v.clone() for k, v in m.state_dict().items()}

        def run():
            m.load_state_dict(sd)          # the running statistics move with every train-mode forward
            return step()
        # the training step of the dilated (non-strided) models does not repeat bit for bit run to run, with or
        # without the audit (measured on an H100 80GB HBM3 at 700 W: BatchNorm parameter gradients move by up to
        # 5e-6 in fp32-grade and 5e-3 in TF32 between identical calls), so only the strided ones are compared
        recs = audited(run, exact=case.strided)
        assert any(r['form'] == ('tf32' if tprec == 'tf32' else '3xtf32') for r in recs), name
    STATE['cases'].add('train')


def test_eval_backward_and_chunked():
    from test_gpu_forward_fp64 import build_model
    x0 = torch.from_numpy(synth.synth_input(3, 40, 17, 2, seed=8)).cuda()
    for strided in (False, True):
        m = build_model(17, [3, 3, 3], 64, strided, False, False).cuda()

        def grads(fwd):
            x = x0.clone().requires_grad_(True)
            m.zero_grad(set_to_none=True)
            y = fwd(x)
            (y * y).sum().backward()
            return [y.detach().clone(), x.grad.clone()] + [p.grad.clone() for p in m.parameters()]
        # the dilated model's backward does not repeat bit for bit run to run, with or without the audit (measured on
        # an H100 80GB HBM3 at 700 W: up to 1.2e-4 between identical calls), so only the strided one is compared
        audited(lambda: grads(m), exact=strided)
        # dilated T_out = 14, strided 4: windows of 5 and 3 output frames
        w = 3 if strided else 5
        audited(lambda: grads(lambda x: engine.run_model_chunked(m, x, w)), exact=strided)
        with torch.no_grad():
            audited(lambda: engine.run_model_chunked(m, x0, w).clone())
    STATE['cases'].add('eval_chunked')


# ------------------------------------------------------------------------------------------------------------------
# streams
# ------------------------------------------------------------------------------------------------------------------
def _stream_model(J, causal, ch=64):
    from test_gpu_forward_fp64 import build_model
    return build_model(J, [3, 3, 3], ch, False, causal, False).cuda()


def test_streams():
    from gast_b200.realtime import CausalStream, PoseStream
    for J, causal in ((17, True), (19, False)):
        m = _stream_model(J, causal)
        n = 3
        frames = torch.from_numpy(synth.synth_input(n, 40, J, 2, seed=J)).cuda()

        def run():
            ps = CausalStream(m, n) if causal else PoseStream(m, n)
            out = []
            with torch.no_grad():
                for t in range(30):                       # the 27-frame ring wraps
                    out.append(ps.push(frames[:, t]))
                out.append(ps.push_frames(frames[:, 30:36].contiguous()))
                if not causal:
                    out.append(ps.peek(4))
                out.append(ps.push(frames[[0, 2], 36], streams=[0, 2]))
            return [o[0] if isinstance(o, tuple) else o for o in out]
        audited(run)
    STATE['cases'].add('streams')


def test_graphed_pool_warm_up():
    from gast_b200.realtime import GraphedPoseStream
    J = 19
    m = _stream_model(J, False)
    frames = torch.from_numpy(synth.synth_input(2, 12, J, 2, seed=3)).cuda()
    skips0 = STATE['skips']

    def run():
        gs = GraphedPoseStream(m, 2, K=2)
        with torch.no_grad():
            return [gs.push(frames[:, 2 * t:2 * t + 2].contiguous())[0] for t in range(5)]
    audited(run, cores=(0,))
    assert STATE['skips'] > skips0, 'no launch ran under capture'
    STATE['cases'].add('graphed')


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
        seen[(r['core'], r['epi'])] += 1
        seen['form:' + r['form']] += 1
        for t in r['shape']:
            seen[t] += 1
        w = worst[(r['core'], r['form'], r['epi'])]
        w[0], w[1], w[2] = max(w[0], r['worst']), max(w[1], r['l2']), w[2] + 1
    lines = ['# %s: %d launches audited, %d skipped under capture\n' % (_card(), len(recs), STATE['skips'])]
    lines += ['# %-28s %d\n' % (k if isinstance(k, str) else '%s/%s' % k, v) for k, v in sorted(seen.items(), key=str)]
    lines += ['# worst %s %s %s: err/bound %.3e l2 %.3e over %d\n' % (k + tuple(v)) for k, v in sorted(worst.items())]
    GA.write_report(lines + [GA.report_line(r) for r in recs])
    print(''.join(lines))
    missing = [k for k in COVERAGE if not seen[k]]
    assert not missing, 'forms no audited launch reached: %s' % missing
