"""The adjoint of the temporal tap gather (seg_adjoint_kernel, csrc/train_kernels.cuh), restated in numpy from the input
side, as the training and gradient backward runs it for every schedule geometry() (csrc/gast_api.cu) builds: the
dilated one (causal or not), the dense ablation, the strided one, and the expand conv (strided inputs whose last
frames no output reads included).  The schedule is restated from the model's own attributes (pad, causal_shift,
filter widths, dense), and checked against its convolution modules.  For every geometry:
  * the gather form (each input element sums its (output frame, tap) terms, residual first, then taps in ascending
    order) equals the scatter form (each output adds into the input frames it read) exactly on small-integer data;
  * every (output frame, tap) pair, and every residual read, is counted exactly once;
  * input frames that no output reads get 0."""
import numpy as np
import pytest

import kinkfree as K


def schedule(m, T, strided_now):
    """(expand, stages) of a forward on clips of T frames, as geometry() decides it.  expand = (T0, s0, k0); a stage is
    (taps, dil, Tin, Tout, tapmap, resmap) with RowMap = (T_out, T_in, t_mul, t_off)."""
    fw = m.filter_widths
    dense = getattr(m, '_gast_dense', False)
    k0 = fw[0]
    s0 = k0 if strided_now else 1
    assert T >= k0
    T0 = (T - k0) // s0 + 1
    stages, Tp, nd = [], T0, k0
    for i in range(1, len(fw)):
        conv = m.layers_conv[2 * (i - 1)]
        if strided_now:
            taps, stride, dil = fw[i], fw[i], 1
            res_mul, res_off = fw[i], (fw[i] // 2 if m._gast_causal else 0) + fw[i] // 2
        else:
            taps, stride, dil = (2 * m.pad[i] + 1, 1, 1) if dense else (fw[i], 1, nd)
            res_mul, res_off = 1, m.pad[i] + m.causal_shift[i]
            # the module convolves with exactly these taps
            assert conv.kernel_size[0] == taps and conv.dilation[0] == dil and conv.stride[0] == 1
        span = (taps - 1) * dil + 1
        assert Tp >= span
        Tn = (Tp - span) // stride + 1
        assert res_off + (Tn - 1) * res_mul < Tp
        stages.append((taps, dil, Tp, Tn, (Tn, Tp, stride, 0), (Tn, Tp, res_mul, res_off)))
        Tp, nd = Tn, nd * fw[i]
    return (T0, s0, k0), stages


def scatter(B, J, Kc, tapmap, taps, dil, src, resmap=None, rsrc=None):
    """the adjoint as the forward's gather reads: output frame t of clip b, tap k adds into input frame
    t*t_mul + t_off + k*dil (np.add.at); returns dX and the number of reads of every input element"""
    T_out, T_in, mul, off = tapmap
    dX = np.zeros((B, T_in, J, Kc), np.float32)
    cnt = np.zeros((B, T_in), np.int64)
    t = np.arange(T_out)
    if rsrc is not None:
        Tr, Tri, rmul, roff = resmap
        assert (Tr, Tri) == (T_out, T_in)
        np.add.at(dX, (slice(None), t * rmul + roff), rsrc)
        np.add.at(cnt, (slice(None), t * rmul + roff), 1)
    for k in range(taps):
        np.add.at(dX, (slice(None), t * mul + off + k * dil), src[:, :, :, k * Kc:(k + 1) * Kc])
        np.add.at(cnt, (slice(None), t * mul + off + k * dil), 1)
    return dX, cnt


def gather(B, J, Kc, tapmap, taps, dil, src, resmap=None, rsrc=None):
    """seg_adjoint_kernel: input frame u sums src over the (t, k) with t*t_mul + t_off + k*dil == u, after the residual
    term; returns dX and the list of (b, t, k) pairs (k = -1: residual) each input frame took"""
    T_out, T_in, mul, off = tapmap
    dX = np.empty((B, T_in, J, Kc), np.float32)
    pairs = []
    for b in range(B):
        for u in range(T_in):
            s = np.zeros((J, Kc), np.float32)
            if rsrc is not None:
                _, _, rmul, roff = resmap
                v = u - roff
                if v >= 0 and v % rmul == 0 and v // rmul < T_out:
                    s = s + rsrc[b, v // rmul]
                    pairs.append((b, v // rmul, -1))
            for k in range(taps):
                v = u - off - k * dil
                if v >= 0 and v % mul == 0 and v // mul < T_out:
                    s = s + src[b, v // mul, :, k * Kc:(k + 1) * Kc]
                    pairs.append((b, v // mul, k))
            dX[b, u] = s
    return dX, pairs


def check(B, J, Kc, tapmap, taps, dil, resmap=None, with_res=False, seed=0):
    T_out, T_in = tapmap[0], tapmap[1]
    rng = np.random.RandomState(seed)
    # small integers (nonzero): every sum is exact in fp32, whatever its order
    src = rng.randint(1, 9, size=(B, T_out, J, taps * Kc)).astype(np.float32)
    rsrc = rng.randint(1, 9, size=(B, T_out, J, Kc)).astype(np.float32) if with_res else None
    ds, cnt = scatter(B, J, Kc, tapmap, taps, dil, src, resmap, rsrc)
    dg, pairs = gather(B, J, Kc, tapmap, taps, dil, src, resmap, rsrc)
    assert np.array_equal(dg, ds)
    # every (output frame, tap) pair once, and every residual read once
    want = {(b, t, k) for b in range(B) for t in range(T_out) for k in range(taps)}
    if with_res:
        want |= {(b, t, -1) for b in range(B) for t in range(T_out)}
    assert len(pairs) == len(set(pairs)) and set(pairs) == want
    # frames no output reads are zero, and only those
    unread = cnt == 0
    assert np.all(dg[unread] == 0) and np.all(dg[~unread] != 0)
    return int(unread.sum()), int((cnt > 1).sum())


CASES = [  # fw, strided model, causal, dense, T
    ([3, 3, 3], False, False, False, 27),
    ([3, 3, 3], False, False, False, 27 + 13),
    ([3, 3, 3], False, True, False, 27),
    ([3, 3, 3], False, True, False, 27 + 13),
    ([3, 3, 3, 3], False, False, False, 81),
    ([3, 3, 3, 3], False, False, False, 81 + 10),
    ([3, 3, 3, 3], False, True, False, 81 + 10),
    ([3, 3, 3], False, False, True, 27),
    ([3, 3, 3], False, False, True, 27 + 13),
    ([3, 3, 3], True, False, False, 27),
    ([3, 3, 3], True, False, False, 27 * 3),
    ([3, 3, 3], True, False, False, 27 * 2 + 2),       # T not a multiple of k0: the last 2 frames are read by no one
    ([3, 3, 3], True, True, False, 27 * 2 + 1),
    ([3, 3, 3, 3], True, False, False, 81 + 4),
]
IDS = ['%s_%s%s%s_T%d' % (''.join(map(str, c[0])), 'strided' if c[1] else 'dilated', '_causal' if c[2] else '',
                          '_dense' if c[3] else '', c[4]) for c in CASES]


def _model(fw, strided, causal, dense):
    return K.module(K.Case(17, fw, 4, 1, 1, strided, causal, dense, True))


def _schedules(m, T, strided):
    """the schedules a call on T frames can take: the model's own, and for a dilated model at T == receptive field
    the strided one its eval-mode forward runs"""
    out = [strided]
    if not strided and not m._gast_dense and T == m.receptive_field():
        out.append(True)
    return out


@pytest.mark.parametrize('fw,strided,causal,dense,T', CASES, ids=IDS)
def test_stage_adjoints(fw, strided, causal, dense, T):
    m = _model(fw, strided, causal, dense)
    B, J = 2, 3
    for sn in _schedules(m, T, strided):
        _, stages = schedule(m, T, sn)
        overlapped = 0
        for i, (taps, dil, Tin, Tout, tapmap, resmap) in enumerate(stages):
            check(B, J, 2, tapmap, taps, dil, resmap, with_res=True, seed=i)
            # the taps alone, and the residual slice alone (the same gather with one tap)
            _, over = check(B, J, 2, tapmap, taps, dil, seed=10 + i)
            overlapped += over
            check(B, J, 2, resmap, 1, 0, seed=20 + i)
        # the taps of different output frames overlap on the dilated and dense schedules, never on the strided one
        assert (overlapped > 0) == (not sn)


@pytest.mark.parametrize('fw,strided,causal,dense,T', CASES, ids=IDS)
def test_expand_adjoint(fw, strided, causal, dense, T):
    m = _model(fw, strided, causal, dense)
    for sn in _schedules(m, T, strided):
        (T0, s0, k0), _ = schedule(m, T, sn)
        conv = m.expand_conv
        if not sn:
            assert conv.kernel_size[0] == k0 and conv.stride[0] == 1
        elif strided:
            assert conv.kernel_size[0] == k0 and conv.stride[0] == k0
        # RowMap{T0, T, s0, 0}, k0 taps one frame apart, Kc = in_features
        unread, over = check(2, 3, m.in_features, (T0, T, s0, 0), k0, 1, seed=T)
        assert unread == 2 * ((T - k0) % s0 if sn else 0)
        assert (over > 0) == (not sn)
