"""fp64 restatement of the device's folded eval forward, with the operands of every tensor-core GEMM rounded to TF32
as the single-pass precision (`gast_set_precision(h, 1)`, `engine.set_precision(model, 'tf32')`) rounds them.

Test infrastructure, CPU only.  The algebra is the one `gast_prepare` and `csrc/gast_api.cu` run, not the reference's
op order (oracle/gast_oracle.py restates that):
  - BatchNorm folded into each conv (the scale into the weight, in fp32 as `fold_conv_kernel` does it);
  - SemCH: one GEMM against [W0 | W1], then the softmax-coefficient mix of the self and neighbour halves;
  - theta / phi collapsed into two row-dots per head (not a GEMM), the `g` convs of all heads one stacked GEMM,
    followed by the attention mix;
  - the block concatenation a 3-segment GEMM, each temporal conv one GEMM over its gathered taps.
Each GEMM the tensor-core core takes (every K segment a multiple of 32, `tc_supported`) gets tf32(A) . tf32(W) when
`rnd` is set; everything else (expand, row-dots, mixes, shrink, GEMMs of other widths) stays fp64.  With `rnd` off
this reproduces the reference's goldens at fp32 rounding level (tests/test_tf32ref_cpu.py).

Activations are channels-last: rows (clip, frame) x joints x channels.  `p` is {state_dict key: fp32 array}.
"""
import numpy as np

from oracle import gast_oracle as O

BN_EPS = np.float32(1e-5)


def tf32(x):
    """cvt.rna.tf32.f32 of fp32(x): round to nearest, ties away from zero, to 10 mantissa bits (the low 13 bits of
    the fp32 pattern cleared).  Inf and NaN pass through.  Returns float32."""
    f = np.ascontiguousarray(x, dtype=np.float32)
    u = f.view(np.uint32)
    finite = (u & np.uint32(0x7F800000)) != np.uint32(0x7F800000)
    r = np.where(finite, (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000), u).astype(np.uint32)
    return r.view(np.float32)


class Gemms(object):
    """the GEMMs of one forward: `rnd` rounds the operands of those the tensor-core core takes; counts them"""

    def __init__(self, rnd):
        self.rnd = rnd
        self.count = 0        # GEMM launches of the device forward
        self.tc = 0           # of them on the tensor-core core

    def __call__(self, A, W, segs):
        """A (..., K) . W (N, K)^T in fp64; segs: the K-segment widths (per tap or concatenated input)"""
        assert sum(segs) == A.shape[-1] == W.shape[1]
        self.count += 1
        if all(k % 32 == 0 for k in segs) and W.shape[0] % 4 == 0:
            self.tc += 1
            if self.rnd:
                A, W = tf32(A), tf32(W)
        return np.asarray(A, np.float64) @ np.asarray(W, np.float64).T


def relu(x):
    return np.maximum(x, 0.0)


def bn_fold(p, pre):
    """(scale, shift) of an eval BatchNorm in fp32, as gast_prepare computes them"""
    s = p[pre + 'weight'].astype(np.float32) / np.sqrt(p[pre + 'running_var'].astype(np.float32) + BN_EPS)
    t = p[pre + 'bias'].astype(np.float32) - p[pre + 'running_mean'].astype(np.float32) * s
    return s, t


def conv_fold(p, wkey, bnpre):
    """conv weight (N, Cin, taps, 1) with the BN scale folded in (fp32) -> (N, taps * Cin) tap-major, and the shift"""
    w = p[wkey].astype(np.float32)
    w = w.reshape(w.shape[0], w.shape[1], -1)
    s, t = bn_fold(p, bnpre)
    wf = (w * s[:, None, None]).astype(np.float32)
    return wf.transpose(0, 2, 1).reshape(w.shape[0], -1), t.astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------
# model/local_attention.py
# ------------------------------------------------------------------------------------------------------------------
def semch_gemm(X, Ws, g):
    """the one SemCH GEMM of a layer: X (R, J, Cin) . [W0 | W1] of every mask's W (2, Cin, Cout) -> per mask
    (X W0, X W1)"""
    Cout = Ws[0].shape[2]
    H = g(X, np.concatenate([w.T for W in Ws for w in W]), [X.shape[-1]])
    return [(H[..., 2 * m * Cout:(2 * m + 1) * Cout], H[..., (2 * m + 1) * Cout:(2 * m + 2) * Cout])
            for m in range(len(Ws))]


def semch_mix(H0, H1, e, mask):
    """SemCHGraphConv's softmax-coefficient mix of the self (H0) and neighbour (H1) products, without BN:
    -> (R, J, Cout).  e (Cout, nnz) or shared (1, nnz), in the mask's row-major nonzero order."""
    Cout = H0.shape[-1]
    J = mask.shape[0]
    rows, cols = np.nonzero(mask)
    adj = np.full((Cout, J, J), -np.inf)
    adj[:, rows, cols] = np.broadcast_to(np.asarray(e, np.float64), (Cout, len(rows)))
    adj = np.exp(adj - adj.max(axis=2, keepdims=True))
    adj /= adj.sum(axis=2, keepdims=True)
    E = np.eye(J)
    return np.einsum('cij,rjc->ric', adj * E, H0) + np.einsum('cij,rjc->ric', adj * (1 - E), H1)


def local_graph(X, p, pre, masks, g):
    """LocalGraph: X (R, J, C) -> (R, J, C)"""
    C = X.shape[-1]
    H = semch_gemm(X, [p[pre + 'gcn_sym.W'], p[pre + 'gcn_con.W']], g)
    outs = []
    for m, (gp, bp) in enumerate((('gcn_sym.', 'bn_1.'), ('gcn_con.', 'bn_2.'))):
        s, t = bn_fold(p, pre + bp)
        y = semch_mix(H[m][0], H[m][1], p[pre + gp + 'e'], masks[m])
        outs.append(relu(y * s + t))
    W, b = conv_fold(p, pre + 'cat_conv.weight', pre + 'cat_bn.')
    return relu(g(np.concatenate(outs, -1), W, [2 * C]) + b)


# ------------------------------------------------------------------------------------------------------------------
# model/global_attention.py
# ------------------------------------------------------------------------------------------------------------------
def _attention(X, p, hp):
    """softmax(LeakyReLU(theta_i . wc_a + phi_j . wc_b)) + C_k from the collapsed row-dots: X (R, J, C) -> (R, J, J)"""
    f64 = lambda k: p[hp + k].astype(np.float64)   # noqa: E731
    wt, wp = f64('theta.weight')[:, :, 0], f64('phi.weight')[:, :, 0]
    wc = f64('concat_project.0.weight').reshape(-1)
    Ci = wt.shape[0]
    a = X @ (wc[:Ci] @ wt) + wc[:Ci] @ f64('theta.bias')
    b = X @ (wc[Ci:] @ wp) + wc[Ci:] @ f64('phi.bias')
    f = a[:, :, None] + b[:, None, :]
    f = np.where(f >= 0, f, 0.2 * f)
    f = np.exp(f - f.max(axis=-1, keepdims=True))
    return f / f.sum(axis=-1, keepdims=True) + f64('C_k')[None]


def global_heads(X, p, prefixes, g):
    """the attention-mixed `g` of the heads at `prefixes` (one stacked GEMM): X (R, J, C) -> (R, J, heads * Cg)"""
    C = X.shape[-1]
    Wg = np.concatenate([p[hp + 'g.weight'][:, :, 0] for hp in prefixes]).astype(np.float32)
    bg = np.concatenate([p[hp + 'g.bias'] for hp in prefixes]).astype(np.float64)
    G = g(X, Wg, [C]) + bg
    Cg = Wg.shape[0] // len(prefixes)
    return np.concatenate([_attention(X, p, hp) @ G[..., h * Cg:(h + 1) * Cg] for h, hp in enumerate(prefixes)], -1)


def global_graph(X, p, pre, g):
    """GlobalGraph (one head): X (R, J, C) -> (R, J, Cg)"""
    return global_heads(X, p, [pre], g)


def multi_global_graph(X, p, pre, g):
    """MultiGlobalGraph: X (R, J, C) -> (R, J, C)"""
    heads = 0
    while (pre + 'attentions.%d.C_k' % heads) in p:
        heads += 1
    Y = global_heads(X, p, [pre + 'attentions.%d.' % h for h in range(heads)], g)
    W, b = conv_fold(p, pre + 'cat_conv.weight', pre + 'cat_bn.')
    return relu(g(Y, W, [Y.shape[-1]]) + b)


# ------------------------------------------------------------------------------------------------------------------
# model/gast_net.py
# ------------------------------------------------------------------------------------------------------------------
def block(X, p, pre, masks, g):
    """GraphAttentionBlock: X (R, J, C) -> (R, J, 2C)"""
    C = X.shape[-1]
    L = local_graph(X, p, pre + 'local_graph_layer.', masks, g)
    Gl = multi_global_graph(X, p, pre + 'global_graph_layer.', g)
    W, b = conv_fold(p, pre + 'cat_conv.weight', pre + 'cat_bn.')
    return relu(g(np.concatenate([X, L, Gl], -1), W, [C, C, C]) + b)


def _blocks(h, p, pre, masks, g):
    B, T, J, C = h.shape
    return block(h.reshape(B * T, J, C), p, pre, masks, g).reshape(B, T, J, 2 * C)


def forward(x, p, masks, filter_widths, causal=False, strided=False, dense=False, rnd=True):
    """the eval forward x (B, T, J, F) -> (y (B, T_out, J, 3) fp64, Gemms).  `strided` is the schedule run
    (Optimized1f, or a dilated model on one receptive field); masks = (sym, con) boolean (J, J)."""
    g = Gemms(rnd)
    fw = list(filter_widths)
    pad, shift, stages = O.model_geometry(fw, causal, strided, dense)
    x = np.asarray(x, np.float64)
    k0 = fw[0]
    s0 = k0 if strided else 1
    T0 = (x.shape[1] - k0) // s0 + 1
    si, ti = bn_fold(p, 'init_bn.')
    xn = x * si + ti
    w = p['expand_conv.weight'].astype(np.float64)[:, :, :, 0]           # (C, F, k0)
    h = sum(xn[:, kk: kk + (T0 - 1) * s0 + 1: s0] @ w[:, :, kk].T for kk in range(k0))
    se, te = bn_fold(p, 'expand_bn.')
    h = _blocks(relu(h * se + te), p, 'layers_graph_conv.0.', masks, g)
    for i, sg in enumerate(stages):
        k, st, dil = sg['k'], sg['stride'], sg['dilation']
        Tp, Cw = h.shape[1], h.shape[3]
        Tn = (Tp - ((k - 1) * dil + 1)) // st + 1
        if strided:
            res = h[:, shift[i + 1] + fw[i + 1] // 2:: fw[i + 1]][:, :Tn]
        else:
            res = h[:, pad[i + 1] + shift[i + 1]:][:, :Tn]
        A = np.concatenate([h[:, tap * dil: tap * dil + (Tn - 1) * st + 1: st] for tap in range(k)], -1)
        Wt, bt = conv_fold(p, 'layers_conv.%d.weight' % (2 * i), 'layers_bn.%d.' % (2 * i))
        tmp = relu(g(A, Wt, [Cw] * k) + bt)
        W1, b1 = conv_fold(p, 'layers_conv.%d.weight' % (2 * i + 1), 'layers_bn.%d.' % (2 * i + 1))
        h = relu(g(tmp, W1, [Cw]) + b1) + res
        h = _blocks(h, p, 'layers_graph_conv.%d.' % (i + 1), masks, g)
    ws = p['shrink.weight'].astype(np.float64).reshape(3, -1)
    return h @ ws.T, g


def module_forward(kind, x, p, masks, rnd=True):
    """the sub-module kinds in their own layouts (as the reference modules take them) -> (y fp64, Gemms):
    'block' (B, C, T, J) -> (B, 2C, T, J); 'local', 'mglobal' (B, T, J, C) -> same; 'global' (BT, C, J) -> (BT, Cg, J);
    'semch' / 'semgc' (B, T, J, Cin) -> (B, T, J, Cout), masks then the single (J, J) mask."""
    g = Gemms(rnd)
    if kind == 'block':
        X = np.asarray(x, np.float64).transpose(0, 2, 3, 1)
        B, T, J, C = X.shape
        return block(X.reshape(B * T, J, C), p, '', masks, g).reshape(B, T, J, -1).transpose(0, 3, 1, 2), g
    if kind == 'global':
        X = np.asarray(x, np.float64).transpose(0, 2, 1)
        return global_graph(X, p, '', g).transpose(0, 2, 1), g
    X = np.asarray(x, np.float64)
    B, T, J, C = X.shape
    X = X.reshape(B * T, J, C)
    if kind == 'local':
        y = local_graph(X, p, '', masks, g)
    elif kind == 'mglobal':
        y = multi_global_graph(X, p, '', g)
    elif kind in ('semch', 'semgc'):
        (H0, H1), = semch_gemm(X, [p['W']], g)
        y = semch_mix(H0, H1, p['e'], masks)
        if 'bias' in p:
            y = y + p['bias'].astype(np.float64)
    else:
        raise ValueError(kind)
    return y.reshape(B, T, J, -1), g
