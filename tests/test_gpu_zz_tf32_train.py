"""GPU: the opt-in TF32 training precision (`gast_set_train_precision(h, 1)`, `engine.set_training_precision(m, 'tf32')`)
and its TF32 weight-gradient kernel (csrc/wgrad_tc.cuh).

  1. single contractions through gast_debug_wgrad against tests/tf32wgradref.py: every dense_tn shape of the
     27f/128ch and 81f/64ch steps at b = 128, ragged and very long M, one to many splits; bitwise repeatable; shapes the
     kernel does not take equal the FFMA kernel bit for bit.  (Repeatability across CUDA-graph replays is checked on
     the whole graphed training step, test_convergence_and_graph_replay.)
  2. every gradient tensor of every tests/kinkfree.py case against fp64 autograd of the torch-CPU port, with the
     number of weight gradients that ran on the new kernel.
  3. switching back to fp32-grade leaves nothing behind.
  4. a student learns a teacher's poses in both precisions (GraphedTrainer + FusedAdam(amsgrad)).
  5. refusals and launch counts.
Measured values go to $GAST_TEST_REPORT_DIR/tf32_train.txt when that is set.
"""
import copy
import os

import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth
import kinkfree as KF
import tf32wgradref as W

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')

# Bars, with the worst values measured on an H100 80GB HBM3 (400 W power limit), one run.
# Single contractions: relative L2 to the emulation (fp32 accumulation against exact sums of the same rounded products;
# measured at most 4.2e-7) and the ratio of the distance to exact fp64 over the distance to the emulation (measured at
# least 710).
WG_L2_BAR = 2e-5
WG_RATIO = 10.0
# Whole models against the fp64 port.  y: the inference TF32 bar (measured 3.5e-3 of max |y|); loss (7.2e-5); every
# gradient tensor in relative L2 (dL/dx at most 4.6e-3, the tensors outside the logit family below at most 7.8e-3).
# The logit family of an attention head, theta.weight, phi.weight and concat_project.0.weight: each gradient is the
# head's logit gradients (a sum that nearly cancels: softmax gradients sum to zero along each row) weighted by the
# input or by theta / phi, so its error follows the terms, not the result, as for theta.bias / phi.bias
# (kinkfree.errors scales those).  In addition the test points keep every LeakyReLU logit only 2.9e-4 - 1.6e-3 of the
# logits' standard deviation from the kink, under the ~1e-3 relative displacement of a TF32 forward, so a few logits
# change slope.  (The widest gap near the median of thousands of logits is that narrow whatever the seed;
# kinkfree.MARGIN's 1e-4 is met, 2e-2 cannot be.)  Measured 6.3e-2, in the case with the narrowest margin.
# Tensors that are zero by construction come out at the rounding level of their terms: measured 2.1e-4 of the
# largest gradient entry (against 1e-6 at fp32 grade).
Y_BAR = 5e-3
LOSS_BAR = 5e-4
GRAD_L2_BAR = 1.5e-2
LOGIT_W_L2_BAR = 1e-1
LOGIT_FAMILY = ('.theta.weight', '.phi.weight', '.concat_project.0.weight')
ZERO_BAR = 1e-3


def report(line):
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        with open(os.path.join(REPORT_DIR, 'tf32_train.txt'), 'a') as f:
            f.write(line + '\n')


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _wgrad(dz, a, core, tc_mode):
    M, N = dz.shape
    K = a.shape[1]
    out = torch.full((N, K), float('nan'), dtype=torch.float32, device='cuda')
    lib = _lib.load()
    rc = lib.gast_debug_wgrad(dz.data_ptr(), a.data_ptr(), out.data_ptr(), M, N, K, core, tc_mode, 0, None,
                              torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return out.cpu().numpy()


def step_shapes(C, fw, J, B, T):
    """(M, N, K) of every dense_tn of one training step of the strided (Optimized1f) model"""
    out = []
    L = len(fw)
    F = B * (T // fw[0])
    KP = -(-fw[0] * 2 // 8) * 8
    out.append((F * J, C, KP))                                    # expand
    for i in range(L):
        Cb = C << i
        if i:
            F //= fw[i]
            out += [(F * J, Cb, Cb), (F * J, Cb, fw[i] * Cb)]    # stage 1x1, stage taps
        out += [(F * J, 2 * Cb, 3 * Cb), (F * J, Cb, Cb), (F * J, Cb, Cb), (F * J, 8, Cb), (F * J, Cb, 2 * Cb),
                (F * J, 4 * Cb, Cb)]
    return out


SHAPES = sorted(set(step_shapes(128, [3, 3, 3], 17, 128, 27) + step_shapes(64, [3, 3, 3, 3], 17, 128, 81) +
                    [(1, 32, 32), (31, 64, 96), (1000, 160, 480), (4097, 1536, 1536), (626688, 128, 128),
                     (700001, 64, 256)]))


@pytest.mark.parametrize('M,N,K', SHAPES)
def test_single_contraction(M, N, K):
    rs = np.random.RandomState((M * 7 + N * 3 + K) % 2 ** 31)
    dZ = rs.standard_normal((M, N)).astype(np.float32)
    A = np.abs(rs.standard_normal((M, K))).astype(np.float32)     # ReLU-like activations
    dz, a = torch.from_numpy(dZ).cuda(), torch.from_numpy(A).cuda()
    ffma = _wgrad(dz, a, 1, 0)
    tc = _wgrad(dz, a, 0, 1)
    tc2 = _wgrad(dz, a, 0, 1)
    assert np.array_equal(tc.view(np.uint32), tc2.view(np.uint32))
    if not W.takes(N, K):
        assert np.array_equal(tc.view(np.uint32), ffma.view(np.uint32))
        return
    emu = W.wgrad(dZ, A, _sms()).astype(np.float64)
    exact = dZ.astype(np.float64).T @ A.astype(np.float64)
    l2 = lambda d, r: float(np.linalg.norm(d) / np.linalg.norm(r))   # noqa: E731
    e_emu, e_exact = l2(tc - emu, emu), l2(tc - exact, exact)
    S, _ = W.split(M, N, K, _sms())
    report('wgrad M=%d N=%d K=%d S=%d: l2 vs emulation %.2e, vs fp64 %.2e (ratio %.0f); ffma vs fp64 %.2e'
           % (M, N, K, S, e_emu, e_exact, e_exact / max(e_emu, 1e-30), l2(ffma - exact, exact)))
    assert e_emu <= WG_L2_BAR, e_emu
    assert e_exact >= WG_RATIO * e_emu, (e_exact, e_emu)


def test_refusals():
    lib = _lib.load()
    z = torch.zeros(64, 32, device='cuda')
    o = torch.zeros(32, 32, device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    assert lib.gast_debug_wgrad(z.data_ptr(), z.data_ptr(), o.data_ptr(), 64, 32, 32, 0, 0, 0, None, st) != 0
    assert 'fp32-grade' in _lib.last_error()
    m = KF.module(KF.CASES['o1f_j16_c16_train']).cuda()
    with pytest.raises(engine.GastError):
        engine.set_training_precision(m, 'bf16')
    m(KF.inputs(KF.CASES['o1f_j16_c16_train']).cuda())
    h = list(m.__dict__['_gast_handles'].values())[0]
    assert h.lib.gast_set_train_precision(h.h, 2) != 0
    assert h.lib.gast_set_train_precision(h.h, -1) != 0
    # inference TF32 alone still refuses training; with the training precision at TF32 it trains
    engine.set_precision(m, 'tf32')
    with pytest.raises(engine.GastError, match='inference-only'):
        m(KF.inputs(KF.CASES['o1f_j16_c16_train']).cuda())
    engine.set_training_precision(m, 'tf32')
    assert engine.get_training_precision(m) == 'tf32' and engine.get_training_precision(m.layers_conv[0]) == 'tf32'
    m(KF.inputs(KF.CASES['o1f_j16_c16_train']).cuda()).sum().backward()
    assert engine.get_training_precision(copy.deepcopy(m)) == 'tf32'
    assert all('precision' not in k for k in m.state_dict())


# ------------------------------------------------------------------------------------------------------------------
# whole-model gradients against fp64
# ------------------------------------------------------------------------------------------------------------------
def _taps(case, m, i):
    if case.strided or not case.dense:
        return case.fw[i]
    return 2 * m.pad[i] + 1


def expected_wgrad_tc(case, m):
    """weight gradients of one backward of `case` that the TF32 kernel takes"""
    n = 0
    for i in range(len(case.fw)):
        Cb = case.ch << i
        n += sum(W.takes(N, K) for N, K in ((2 * Cb, 3 * Cb), (Cb, Cb), (Cb, Cb), (8, Cb), (Cb, 2 * Cb), (4 * Cb, Cb)))
        if i:
            n += W.takes(Cb, Cb) + W.takes(Cb, _taps(case, m, i) * Cb)
    return n


def _run(case, ref, frozen):
    m = KF.module(case)
    m.load_state_dict(ref['sd'])
    m = m.cuda().train(case.training).requires_grad_(not frozen)
    engine.set_training_precision(m, 'tf32')
    x = ref['x'].cuda().requires_grad_()
    y = m(x)
    loss = torch.mean(torch.norm(y - ref['target'].cuda(), dim=3))
    loss.backward()
    got = {} if frozen else {k: p.grad.cpu().double() for k, p in m.named_parameters()}
    got['x'] = x.grad.cpu().double()
    h = list(m.__dict__['_gast_handles'].values())[0]
    return y.detach().cpu().double(), float(loss), got, h.wgrad_tc_launches(), m


@pytest.mark.parametrize('name', sorted(KF.CASES))
def test_every_gradient_vs_fp64_port(name):
    case = KF.CASES[name]
    ref = KF.reference(name)
    relu, leaky, _ = ref['margins']
    y, loss, got, n_tc, m = _run(case, ref, frozen=False)
    y_err = (y - ref['y']).abs().max().item() / ref['y'].abs().max().item()
    loss_err = abs(loss - ref['loss']) / abs(ref['loss'])
    err = KF.errors(got, ref['grads'], ref['scales'])
    worst = max((v for v in err.items() if v[1][0] is not None), key=lambda t: t[1][0])
    rest = max((v for v in err.items() if v[1][0] is not None and not v[0].endswith(LOGIT_FAMILY)),
               key=lambda t: t[1][0])
    zero = max((v[1] for v in err.values() if v[0] is None), default=0.0)
    _, _, frozen, n_tc_frozen, _ = _run(case, ref, frozen=True)
    want = expected_wgrad_tc(case, m)
    total = 6 * len(case.fw) + 2 * (len(case.fw) - 1) + 1
    report('%s: y %.2e loss %.2e | worst l2 %.2e %s | other tensors %.2e %s | dx l2 %.2e | zero %.1e | margins %.1e '
           '%.1e | weight gradients on the TF32 kernel %d of %d' % (name, y_err, loss_err, worst[1][0], worst[0],
                                                                   rest[1][0], rest[0], err['x'][0], zero, relu, leaky,
                                                                   n_tc, total))
    assert n_tc == want, (n_tc, want)
    assert n_tc_frozen == 0
    if case.ch >= 128:
        assert n_tc > total / 2
    assert y_err <= Y_BAR, y_err
    assert loss_err <= LOSS_BAR, loss_err
    bar = lambda k: LOGIT_W_L2_BAR if k.endswith(LOGIT_FAMILY) else GRAD_L2_BAR   # noqa: E731
    bad = [(k, l2) for k, (l2, mx) in err.items() if l2 is not None and l2 > bar(k)]
    assert not bad, bad
    assert zero <= ZERO_BAR, zero
    dx_l2 = float((frozen['x'] - ref['grads']['x']).norm() / ref['grads']['x'].norm())
    assert dx_l2 <= GRAD_L2_BAR, dx_l2


# ------------------------------------------------------------------------------------------------------------------
# nothing leaks into fp32-grade
# ------------------------------------------------------------------------------------------------------------------
def _step(m, x, tgt):
    xx = x.clone().requires_grad_()
    for p in m.parameters():
        p.grad = None
    y = m(xx)
    torch.mean(torch.norm(y - tgt, dim=3)).backward()
    return [y.detach().clone(), xx.grad.clone()] + [p.grad.clone() for p in m.parameters()]


def test_switch_back_leaves_nothing():
    """a TF32 training step and a TF32 eval backward on a handle, then fp32-grade again: bitwise the results of a
    model that was never switched"""
    case = KF.CASES['o1f_j17_c128_train']
    x = KF.inputs(case).cuda()
    base = KF.module(case).cuda()
    sd = copy.deepcopy(base.state_dict())
    with torch.no_grad():
        tgt = torch.zeros_like(base.eval()(x))
    fresh, used = copy.deepcopy(base), copy.deepcopy(base)
    for train in (True, False):
        fresh.train(train)
        used.train(train)
        engine.set_training_precision(used, 'tf32')
        _step(used, x, tgt)
        engine.set_training_precision(used, 'fp32')
        used.load_state_dict(sd)
        a, b = _step(fresh, x, tgt), _step(used, x, tgt)
        for u, v in zip(a, b):
            assert torch.equal(u, v), train
        fresh.load_state_dict(sd)
        used.load_state_dict(sd)


# ------------------------------------------------------------------------------------------------------------------
# convergence, graph replay, launch counts
# ------------------------------------------------------------------------------------------------------------------
def _student_teacher_losses(prec, core, steps=200, every=20, check_replay=False):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModelOptimized1f
    from gast_b200.pipeline import FusedAdam
    from gast_b200.trainer import GraphedTrainer
    J, b, T = 17, 128, 27
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    teacher = SpatioTemporalModelOptimized1f(adj, J, 2, J, [3, 3, 3], channels=64, dropout=0.0)
    synth.randomize_module(teacher, 101)
    teacher = teacher.cuda().eval()
    student = SpatioTemporalModelOptimized1f(adj, J, 2, J, [3, 3, 3], channels=64, dropout=0.0)
    synth.randomize_module(student, 202)
    student = student.cuda()
    engine.set_training_precision(student, prec)
    engine.set_gemm_core(core)
    try:
        xs = [torch.from_numpy(synth.synth_input(b, T, J, 2, seed=1000 + i)).cuda() for i in range(8)]
        with torch.no_grad():
            ys = [teacher(x) for x in xs]
        tr = GraphedTrainer(student, lambda ps: FusedAdam(ps, lr=1e-3, amsgrad=True), (b, T, J, 2), (b, 1, J, 3))
        out = []
        replay_ok = None
        for s in range(steps):
            x, y = xs[s % 8], ys[s % 8]
            if check_replay and s == 5:
                # the graph replay's gradients against an eager forward + backward of the same step
                tr.x.copy_(x)
                tr.y.copy_(y)
                tr.y[:, :, 0] = 0
                tr.graph.replay()
                g_graph = tr.flat.flat.clone()
                tr.flat.zero_()
                sd = copy.deepcopy(student.state_dict())
                loss = torch.mean(torch.norm(student(tr.x) - tr.y, dim=3))
                loss.backward()
                g_eager = tr.flat.flat.clone()
                student.load_state_dict(sd)
                replay_ok = torch.equal(g_graph, g_eager)
            loss = tr.step(x, y)
            if s % every == 0 or s == steps - 1:
                out.append(float(loss))
        h = list(student.__dict__['_gast_handles'].values())[0]
        return out, replay_ok, h.launches(), h.wgrad_tc_launches()
    finally:
        engine.set_gemm_core(0)


def test_convergence_and_graph_replay():
    tf, replay_ok, n_tf, ntc_tf = _student_teacher_losses('tf32', 0, check_replay=True)
    fp, _, n_fp, ntc_fp = _student_teacher_losses('fp32', 0)
    ff, _, _, _ = _student_teacher_losses('fp32', 1)
    spread = max(abs(a - b) / b for a, b in zip(fp, ff))
    dev = max(abs(a - b) / b for a, b in zip(tf, fp))
    report('convergence: tf32 %s' % ' '.join('%.4f' % v for v in tf))
    report('convergence: fp32 %s' % ' '.join('%.4f' % v for v in fp))
    report('convergence: fp32 ffma %s' % ' '.join('%.4f' % v for v in ff))
    report('convergence: fp32 tc-vs-ffma spread %.3e, tf32 vs fp32 %.3e; launches per step fp32 %d (%d on the TF32 '
           'weight-gradient kernel), tf32 %d (%d)' % (spread, dev, n_fp, ntc_fp, n_tf, ntc_tf))
    assert tf[-1] <= 0.5 * tf[0] and fp[-1] <= 0.5 * fp[0], (tf, fp)
    assert dev <= max(0.05, 3 * spread), (dev, spread)
    assert replay_ok
    assert ntc_fp == 0 and ntc_tf == 3 * 5 + 2 * 2
    assert n_tf == n_fp
