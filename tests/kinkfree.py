"""Kink-free test points for exact gradient checks.

Every ReLU of the lifting network follows a BatchNorm and every attention head passes its logits through
LeakyReLU(0.2).  At an arbitrary (synthetic) test point some of those inputs sit within fp32 rounding of zero, so an
fp32 run can land on the other side of a kink and take a discretely different gradient path: fp64 then stops being
a reference, and the gradient checks have to be written around that noise.

`make_kink_free` moves every kink threshold into a gap of the fp64 pre-activations, layer by layer in forward order
(each step leaves every earlier layer unchanged):
  * ReLU after a BatchNorm: the BatchNorm output is gamma * zhat + beta, and zhat does not depend on beta (batch or
    running statistics alike).  Per channel, beta is set so that -beta/gamma falls in the widest gap of that
    channel's zhat values near their median: about half of each channel stays active.
  * LeakyReLU logits a_i + b_j of a head: shifted through theta.bias along the theta half of concat_project's
    weight, so that zero falls in the widest gap near the median of the head's logits: both slopes stay in use (on
    one linear piece softmax would cancel a_i, and every theta.* gradient would vanish).
There the network is smooth in a neighbourhood much wider than fp32 rounding, fp64 autograd of the torch-CPU port
(oracle/gast_torch_ref.py) is an exact reference, and every gradient tensor can be held to rounding-level bars.
"""
import functools
from collections import namedtuple

import numpy as np
import torch

from gast_b200 import synth
import dropoutref as D

# drop: the dropout probability of the module (train-mode cases replay the library's masks, see `drop_masks`)
Case = namedtuple('Case', 'J fw ch B T strided causal dense training drop', defaults=(0.0,))

DROP_SEED = 61    # torch.manual_seed of every dropout forward at a kink-free point: it fixes the library's masks

WINDOW = (0.3, 0.7)    # quantile window around the median in which the widest gap is chosen


def masks(J):
    from oracle import gast_oracle as O
    return tuple(torch.from_numpy(a) for a in O.local_masks(O.adj_from_parents(synth.skeleton_parents(J))))


def module(case, seed=5):
    """the drop-in module of `case` with synthetic weights and the case's dropout, in the case's mode"""
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    J = case.J
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    if case.strided:
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, case.fw, causal=case.causal, dropout=case.drop,
                                            channels=case.ch)
    else:
        m = SpatioTemporalModel(adj, J, 2, J, case.fw, causal=case.causal, dropout=case.drop, channels=case.ch,
                                dense=case.dense)
    synth.randomize_module(m, seed)
    return m.train(case.training)


_MASKS = {}


def drop_masks(case):
    """the scaled dropout masks (dropoutref.masks) a training forward of `case` draws right after
    torch.manual_seed(DROP_SEED); None without dropout"""
    if not (case.training and case.drop > 0):
        return None
    key = repr(case)
    if key not in _MASKS:
        _MASKS[key] = D.masks(case, case.B, case.T, case.J, case.drop, D.engine_seed(DROP_SEED))
    return _MASKS[key]


def port_forward(p, x, case, tap=None, drop=None, stats=None):
    """the port's forward of `case`; `drop`: the dropout masks to apply (dropoutref.masks), by default the case's own
    (drop_masks)"""
    from oracle import gast_torch_ref as TR
    drop = drop_masks(case) if drop is None else drop
    return TR.forward(x, p, masks(case.J), case.fw, causal=case.causal, strided=case.strided, dense=case.dense,
                      training=case.training, stats=stats, drop=0.0 if drop is None else D.dropper(drop), tap=tap)


def _gap_threshold(v):
    """rows of v (R, n): the midpoint of the widest gap between consecutive sorted values inside the quantile WINDOW"""
    s, _ = torch.sort(v, dim=1)
    n = s.shape[1]
    lo, hi = int(WINDOW[0] * (n - 1)), max(int(WINDOW[1] * (n - 1)), int(WINDOW[0] * (n - 1)) + 1)
    d = s[:, lo + 1:hi + 1] - s[:, lo:hi]
    i = torch.argmax(d, dim=1, keepdim=True)
    return 0.5 * (torch.gather(s[:, lo:hi], 1, i) + torch.gather(s[:, lo + 1:hi + 1], 1, i)).squeeze(1)


class _Stop(Exception):
    pass


def _is_head(p, name):
    return (name + 'concat_project.0.weight') in p


def make_kink_free(sd, x, case, drop=None):
    """state_dict `sd` (name -> tensor) -> a copy whose BatchNorm biases and theta biases put every kink of the
    forward at `x` (in the case's mode, with the dropout masks `drop` as in port_forward) into a gap of the fp64
    pre-activations.  Returns (new state_dict in the dtypes of `sd`, margins as returned by `margins`)."""
    p = {k: (v.detach().double().clone() if v.dtype.is_floating_point else v.clone()) for k, v in sd.items()}
    xd = x.detach().double()
    done = set()

    def place(name, h):
        if name in done:
            return
        done.add(name)
        if _is_head(p, name):
            w = p[name + 'concat_project.0.weight'].reshape(-1)
            wt = w[:w.numel() // 2]                          # the theta half: logits a_i + b_j, a = wt . theta_i
            t = _gap_threshold(h.reshape(1, -1))[0]
            p[name + 'theta.bias'] -= t * wt / wt.dot(wt)    # every logit moves by -t
        else:
            gamma, beta = p[name + 'weight'], p[name + 'bias']
            C = h.shape[1]
            zhat = (h.transpose(0, 1).reshape(C, -1) - beta[:, None]) / gamma[:, None]
            beta.copy_(-gamma * _gap_threshold(zhat))
        raise _Stop                                          # the layers after this one have to see the new value

    with torch.no_grad():
        while True:
            try:
                port_forward(p, xd, case, tap=place, drop=drop)
                break
            except _Stop:
                pass
    out = {k: v.to(sd[k].dtype) for k, v in p.items()}
    return out, margins(out, x, case, drop)


def margins(sd, x, case, drop=None):
    """in fp64 at `x`: (min over BatchNorm channels of min |ReLU input| / std of that channel's ReLU input,
    min over heads of min |logit| / std of the head's logits, {kink name: its margin})"""
    p = {k: (v.detach().double() if v.dtype.is_floating_point else v) for k, v in sd.items()}
    per = {}

    def tap(name, h):
        if _is_head(p, name):
            v = h.reshape(1, -1)
        else:
            v = h.transpose(0, 1).reshape(h.shape[1], -1)
        per[name] = float((v.abs().min(dim=1).values / v.std(dim=1)).min())

    with torch.no_grad():
        port_forward(p, x.detach().double(), case, tap=tap, drop=drop)
    relu = min(v for k, v in per.items() if not _is_head(p, k))
    leaky = min(v for k, v in per.items() if _is_head(p, k))
    return relu, leaky, per


def inputs(case, seed=3):
    """synthetic keypoints (B, T, J, 2) for `case`"""
    return torch.from_numpy(synth.synth_input(case.B, case.T, case.J, 2, seed=seed))


def target(y_shape, seed=4):
    return torch.from_numpy((0.5 * np.random.RandomState(seed).standard_normal(tuple(y_shape))).astype(np.float32))


def port_grads(sd, x, tgt, case, dtype, drop=None):
    """y, loss, every gradient (by parameter name, 'x' for dL/dx) of mpjpe(port(x), tgt) in `dtype`, and the error
    scales of the bias gradients whose value is a cancelling sum (see `errors`)"""
    from oracle import gast_torch_ref as TR
    p = {k: (v.to(dtype).clone().requires_grad_('running' not in k) if v.dtype.is_floating_point else v)
         for k, v in sd.items()}
    dlogits = {}

    def tap(name, h):
        if _is_head(p, name) and h.requires_grad:
            h.register_hook(lambda g, name=name: dlogits.__setitem__(name, float(g.abs().sum())))

    xx = x.to(dtype).clone().requires_grad_()
    y = port_forward(p, xx, case, tap=tap, drop=drop)
    loss = TR.mpjpe(y, tgt.to(dtype))
    loss.backward()
    g = {k: v.grad.double() for k, v in p.items() if v.grad is not None}
    g['x'] = xx.grad.double()
    scales = {}
    for name, a in dlogits.items():
        w = p[name + 'concat_project.0.weight'].detach().double().reshape(-1)
        for key, half in (('theta.bias', w[:w.numel() // 2]), ('phi.bias', w[w.numel() // 2:])):
            scales[name + key] = (float(half.norm()) * a, float(half.abs().max()) * a)
    return y.detach().double(), float(loss.detach()), g, scales


def errors(got, ref, scales):
    """per tensor: (relative L2 error, max |g - g_ref| / max |g_ref|) of `got` against `ref`.
    The theta.bias and phi.bias gradients of a head are one scalar times a half of its concat_project weight; that
    scalar is the sum of all of the head's logit gradients, which nearly cancels (softmax gradients sum to zero
    along each row, only the LeakyReLU slopes keep it from zero).  Its rounding error follows the magnitude of the
    terms, not of the sum, so for these two the L2 and max errors are taken relative to (|half| . sum |dL/dlogit|)
    and (max |half| . sum |dL/dlogit|) from `scales`.
    Tensors whose reference is zero by construction (at most 1e-12 of the largest reference entry) map to
    (None, max |g| / largest reference entry)."""
    top = max(float(v.abs().max()) for v in ref.values())
    out = {}
    for k, r in ref.items():
        g = got[k].double()
        if float(r.abs().max()) <= 1e-12 * top:
            out[k] = (None, float(g.abs().max()) / top)
            continue
        l2_den, mx_den = scales.get(k, (float(r.norm()), float(r.abs().max())))
        out[k] = (float((g - r).norm()) / l2_den, float((g - r).abs().max()) / mx_den)
    return out


# The case matrix of tests/test_kinkfree_cpu.py and tests/test_gpu_grad_exact.py.  It reaches the branches of the
# backward kernels: frame tiles of 120, 128, 119 and 114 rows (J = 15, 16, 17, 19); 16 channels (K % 32 != 0: the FFMA
# core runs in any mode, dense_nn pads N to 32), 48 (not a multiple of 32, 96 is: both cores within one step), 128
# (exact tiles), 160 (a ragged second N / K tile of the tensor-core GEMM and of wgrad_tn_kernel); the strided
# Optimized1f model, the dilated model at T = receptive field (the needed-only schedule), dilated causal over a
# whole sequence longer than the receptive field (overlapping taps in seg_scatter_add_kernel), the dense ablation
# and a first filter width of 5; train mode (batch statistics) and eval mode (running statistics).  The `_drop` cases
# train with dropout, on the library's own masks (tests/dropoutref.py): the reference's default p = 0.05, p = 0.5 and
# 0.25, and p = 0.9 (kept values scaled by 10), at the residual, LocalGraph and MultiGlobalGraph sites of the strided,
# dilated, causal (a non-trivial residual frame map), dense and first-width-5 models.  The `_3333` pair is the
# reference's 81-frame four-stage architecture, without and with dropout.  The causal dropout case runs at B = 3: at
# B = 2 its masks make the init_bn.weight gradient a sum whose terms cancel 4000-fold (40- to 400-fold in every other
# case), so the terms' fp32 rounding, ~5e-8 of their size, reaches 2e-4 of the result on both GEMM cores.
CASES = {
    'o1f_j17_c128_train': Case(17, [3, 3, 3], 128, 16, 27, True, False, False, True),
    'o1f_j17_c128_eval': Case(17, [3, 3, 3], 128, 8, 27, True, False, False, False),
    'o1f_j16_c16_train': Case(16, [3, 3, 3], 16, 6, 27, True, False, False, True),
    'o1f_j19_c160_train': Case(19, [3, 3], 160, 8, 9, True, False, False, True),
    'o1f_j19_c160_eval': Case(19, [3, 3], 160, 8, 9, True, False, False, False),
    'dilated_rf_j15_c48_eval': Case(15, [3, 3, 3], 48, 3, 27, False, False, False, False),
    'dilated_rf_j16_c128_train': Case(16, [3, 3, 3], 128, 2, 27, False, False, False, True),
    'causal_T40_j17_c48_train': Case(17, [3, 3, 3], 48, 2, 40, False, True, False, True),
    'causal_T40_j19_c16_eval': Case(19, [3, 3, 3], 16, 2, 40, False, True, False, False),
    'dense_j15_c16_train': Case(15, [3, 3, 3], 16, 2, 28, False, False, True, True),
    'fw5_o1f_j17_c48_train': Case(17, [5, 3], 48, 6, 15, True, False, False, True),
    'fw5_dilated_j16_c32_eval': Case(16, [5, 3], 32, 3, 15, False, False, False, False),
    'o1f_j17_c128_train_drop05': Case(17, [3, 3, 3], 128, 16, 27, True, False, False, True, 0.05),
    'o1f_j19_c160_train_drop50': Case(19, [3, 3], 160, 8, 9, True, False, False, True, 0.5),
    'dilated_rf_j16_c128_train_drop25': Case(16, [3, 3, 3], 128, 2, 27, False, False, False, True, 0.25),
    'causal_T40_j17_c48_train_drop25': Case(17, [3, 3, 3], 48, 3, 40, False, True, False, True, 0.25),
    'dense_j15_c16_train_drop05': Case(15, [3, 3, 3], 16, 2, 28, False, False, True, True, 0.05),
    'fw5_o1f_j17_c48_train_drop90': Case(17, [5, 3], 48, 6, 15, True, False, False, True, 0.9),
    'o1f_j17_c32_3333_train': Case(17, [3, 3, 3, 3], 32, 4, 81, True, False, False, True),
    'o1f_j17_c32_3333_train_drop05': Case(17, [3, 3, 3, 3], 32, 4, 81, True, False, False, True, 0.05),
}

MARGIN = 1e-4   # least |kink input| / std a test point must keep: far above the fp32 / 3xTF32 forward error (~1e-6)


@functools.lru_cache(maxsize=None)
def reference(name):
    """the kink-free test point of CASES[name] and its fp64 reference: dict with the state_dict 'sd', 'x', 'target',
    'margins', and the port's fp64 'y', 'loss', 'grads', 'scales' (with the case's dropout masks, drop_masks)"""
    case = CASES[name]
    x = inputs(case)
    sd, marg = make_kink_free(module(case).state_dict(), x, case)
    with torch.no_grad():
        shape = port_forward({k: (v.double() if v.dtype.is_floating_point else v) for k, v in sd.items()},
                             x.double(), case).shape
    tgt = target(shape)
    y, loss, grads, scales = port_grads(sd, x, tgt, case, torch.float64)
    return dict(sd=sd, x=x, target=tgt, margins=marg, y=y, loss=loss, grads=grads, scales=scales)


# Per-tensor bars of every gradient (relative L2 error; max error relative to the tensor's largest entry), of y
# (max error relative to max |y|) and of the loss (relative), against the fp64 port at the kink-free points.  Each is
# about 4x the worst value measured over CASES on an H100 80GB HBM3 (700 W power limit): per-tensor L2 1.2e-5 and max
# 1.1e-5 on the default ('tc': 3xTF32 tensor cores where the shapes allow, FFMA elsewhere), 2.2e-5 and 2.8e-5 on the
# FFMA core; y 3.5e-6, loss 1.8e-7.  The fp32 torch-CPU port stays within the FFMA bars (tests/test_kinkfree_cpu.py).
# The dropout cases and the four-stage pair, measured on the same card and power limit, stay within a quarter of
# these: per-tensor L2 8.4e-6 and max 1.0e-5 on 'tc', 1.6e-5 and 1.4e-5 on FFMA; y 3.7e-6, loss 1.4e-7.
# The zero-by-construction bar does not: init_bn.bias, the sum of every dL/d(init_bn output), reached 6.9e-7 of the
# largest gradient entry ('tc', o1f_j17_c32_3333_train_drop05; 2.4e-7 without dropout; 1.4e-6 in the fp32 CPU port).
# Its rounding follows the size of the gradient reaching init_bn, which in that case is 4x larger against the largest
# gradient entry than in the three-stage cases (init_bn.weight's gradient is 0.8 of it, not 0.1), so ZERO_BAR is
# about 4x that worst value.
L2_BAR = {'ffma': 1e-4, 'tc': 5e-5}
MAX_BAR = {'ffma': 1.2e-4, 'tc': 5e-5}
Y_BAR = 1.5e-5
LOSS_BAR = 8e-7
ZERO_BAR = 3e-6     # max |g| / largest gradient entry, for a tensor that is zero by construction


def check(got, ref, scales, core):
    """(list of tensors outside the bars of `core` ('tc' or 'ffma'), {tensor: (l2, max)}) for gradients `got`
    against the fp64 `ref`"""
    l2_bar, max_bar = L2_BAR[core], MAX_BAR[core]
    err = errors(got, ref, scales)
    bad = []
    for k, (l2, mx) in err.items():
        if (mx > ZERO_BAR) if l2 is None else (l2 > l2_bar or mx > max_bar):
            bad.append((k, l2, mx))
    return bad, err
