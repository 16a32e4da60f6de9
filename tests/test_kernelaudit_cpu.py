"""CPU checks of the per-launch audit of the expand, row-dot, attention-mix and shrink kernels (tests/kernelaudit.py)
without a GPU.

Launches are laid out in a host address space (HostMemory, fp32 and fp16 buffers) whose reads fail outside a buffer,
so the snapshot is also held to reading only inside the allocations a launch touches; their outputs come from a numpy
emulation of each kernel's fp32 order (the FMA chains of 4 channels per lane, the xor butterfly, the softmax rows).
  * The vectorised fp64 restatement against a per-element loop over the same definitions.
  * The bounds hold for the emulation, in fp32 and with fp16 inputs and outputs, and the fp16 range edge follows
    round to nearest: inf at or above 65520, finite below.
  * Teeth: the checker refuses an output moved by 16 fp32 ulps or 2 fp16 ulps on operands of one sign (S = |y|), an
    expand or shrink row read from the neighbouring frame, a mix whose head h used head h + 1's attention, a value
    written past the owned columns, a loss moved by 16 ulps, and an fp16 overflow on the wrong side of 65520.
"""
import numpy as np
import pytest

import gemmaudit as GA
import kernelaudit as KA

F32, F16 = 0, 1


class HostMemory(object):
    """numpy buffers (float32 or float16) at fake, 256-byte-aligned addresses with gaps between them; a read must stay
    in one buffer and match its type"""

    def __init__(self):
        self.bufs = []
        self.next = 1 << 20

    def add(self, a, t=F32):
        a = np.ascontiguousarray(a, np.float16 if t else np.float32).ravel()
        base = self.next
        self.bufs.append((base, a))
        self.next += ((a.size * a.itemsize + 255) // 256 + 4) * 256
        return base

    def _get(self, ptr, n, dtype):
        for base, a in self.bufs:
            if base <= ptr < base + a.nbytes:
                assert a.dtype == dtype, 'read of %s at 0x%x from a %s buffer' % (dtype, ptr, a.dtype)
                off = (ptr - base) // a.itemsize
                assert (ptr - base) % a.itemsize == 0 and off + n <= a.size, \
                    'read of %d elements at 0x%x runs past its allocation' % (n, ptr)
                return a[off:off + n].astype(np.float32)
        raise AssertionError('read at 0x%x is in no allocation' % ptr)

    def read(self, ptr, n):
        return self._get(ptr, n, np.float32)

    def read16(self, ptr, n):
        return self._get(ptr, n, np.float16)


def record(kind, **kw):
    P = {k: 0 for k in KA.FIELDS + KA.POINTERS}
    P['kind'] = KA.KINDS.index(kind)
    P.update(kw)
    return P


# ------------------------------------------------------------------------------------------------------------------
# numpy emulations of the kernels' fp32 order
# ------------------------------------------------------------------------------------------------------------------
def fma(a, b, c):
    """fp32 fmaf: the exact product (fp32 operands fit a double) plus c, rounded once"""
    return (np.float64(1) * a * b + c).astype(np.float32)


def lane_dot(X, Wt):
    """warp-per-row dot products of X (R, K) with the rows of Wt (Q, K) as rowdot_kernel / shrink_kernel order them:
    lane l chains fmaf(x.x, w.x, fmaf(x.y, w.y, fmaf(x.z, w.z, fmaf(x.w, w.w, acc)))) over k = 4 l + 128 i, then
    the xor butterfly 16, 8, 4, 2, 1 -> (R, Q) float32"""
    R, K = X.shape
    Kp = -(-K // 128) * 128
    Xp = np.zeros((R, Kp), np.float32)
    Xp[:, :K] = X
    Wp = np.zeros((Wt.shape[0], Kp), np.float32)
    Wp[:, :K] = Wt
    Xl = Xp.reshape(R, Kp // 128, 32, 4)
    Wl = Wp.reshape(-1, Kp // 128, 32, 4)
    acc = np.zeros((R, Wt.shape[0], 32), np.float32)
    for it in range(Kp // 128):
        for c in (3, 2, 1, 0):
            acc = fma(Xl[:, None, it, :, c], Wl[None, :, it, :, c], acc)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = (acc + acc[:, :, lanes ^ o]).astype(np.float32)
    return acc[:, :, 0]


def emu_expand(x, We, be):
    v = np.broadcast_to(be, (x.shape[0], be.size)).astype(np.float32)
    for k in range(x.shape[1]):
        v = fma(We[k][None, :], x[:, k:k + 1], v)
    return np.maximum(v, np.float32(0))


def emu_softmax(ab, ck, J, heads):
    """the attention rows (F, heads, J, J) of global_mix_kernel in fp32"""
    ab = ab.reshape(-1, J, 2 * heads)
    a, b = ab[:, :, 0::2].transpose(0, 2, 1), ab[:, :, 1::2].transpose(0, 2, 1)
    s = (a[:, :, :, None] + b[:, :, None, :]).astype(np.float32)
    s = np.where(s >= 0, s, (np.float32(0.2) * s).astype(np.float32))
    v = np.exp((s - s.max(axis=3, keepdims=True)).astype(np.float32)).astype(np.float32)
    tot = np.zeros(v.shape[:3], np.float32)
    for j in range(J):
        tot = (tot + v[..., j]).astype(np.float32)
    inv = (np.float32(1) / tot).astype(np.float32)
    return ((v * inv[..., None]).astype(np.float32) + ck[None]).astype(np.float32)


def emu_mix(G, att, J, heads, Cg, head_of=None):
    F = G.shape[0] // J
    G = G.reshape(F, J, -1)
    Y = np.zeros_like(G)
    for h in range(heads):
        hh = h if head_of is None else head_of(h)
        cs = slice(h * Cg, (h + 1) * Cg)
        o = np.zeros((F, J, Cg), np.float32)
        for j in range(J):
            o = fma(att[:, hh, :, j][:, :, None], G[:, j, cs][:, None, :], o)
        Y[:, :, cs] = o
    return Y.reshape(F * J, -1)


def to16(a):
    return np.asarray(a, np.float32).astype(np.float16).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------
# host launches
# ------------------------------------------------------------------------------------------------------------------
def expand_launch(rs, J=17, B=2, T=None, T0=3, stride=3, taps=3, Fin=2, C=48, tin=F32, tout=F32, positive=False,
                  scale=1.0):
    mem = HostMemory()
    T = T or (T0 - 1) * stride + taps            # the frames the clip's windows reach
    x = rs.standard_normal((B, T, J, Fin)).astype(np.float32)
    KF = taps * Fin
    We = (rs.standard_normal((KF, C)) / np.sqrt(KF)).astype(np.float32)
    be = (0.3 * rs.standard_normal(C)).astype(np.float32)
    if positive:
        x, We, be = np.abs(x) + 0.1, np.abs(We) + 0.1, np.abs(be) + 0.1
    x = (scale * x).astype(np.float32)
    if tin:
        x = to16(x)
    rows = B * T0 * J
    P = record('expand', variant=6 if KF <= 6 else 10, in_type=tin, out_type=tout, rows=rows, K=C, ld=C, J=J, T=T,
               T0=T0, stride=stride, taps=taps, Fin=Fin)
    P['x'] = mem.add(x, tin)
    P['We'], P['be'] = mem.add(We), mem.add(be)
    P['out'] = mem.add(np.full((rows, C), 7.0), tout)
    S = KA.snapshot(P, mem)
    y = emu_expand(S['x'], S['We'], S['be'])
    return P, S, (y.astype(np.float16).astype(np.float32) if tout else y), mem


def dot_launch(rs, kind, R=45, K=160, ld=None, heads=4, tin=F32, tout=F32, positive=False):
    mem = HostMemory()
    ld = ld or K
    X = rs.standard_normal((R, ld)).astype(np.float32)
    Q = 2 * heads if kind == 'rowdot' else 3
    Wt = (rs.standard_normal((Q, K)) / np.sqrt(K)).astype(np.float32)
    cab = (0.2 * rs.standard_normal(Q)).astype(np.float32)
    if positive:
        X, Wt, cab = np.abs(X) + 0.1, np.abs(Wt) + 0.01, np.abs(cab)
    if tin:
        X = to16(X)
    P = record(kind, in_type=tin, out_type=tout, rows=R, K=K, ld=ld, heads=heads if kind == 'rowdot' else 0,
               variant=2 * heads if kind == 'rowdot' else 0)
    P['x'] = mem.add(X, tin)
    if kind == 'rowdot':
        P['U'], P['cab'] = mem.add(Wt), mem.add(cab)
        P['ab'] = mem.add(np.full((R, Q), 7.0))
    else:
        P['Ws'] = mem.add(Wt)
        P['out'] = mem.add(np.full((R, 3), 7.0), tout)
    target = None
    if kind == 'shrink_mpjpe':
        target = rs.standard_normal((R, 3)).astype(np.float32)
        P['target'] = mem.add(target)
        P['loss'] = mem.add(np.zeros(1))
    S = KA.snapshot(P, mem)
    y = lane_dot(S['X'], S['U'] if kind == 'rowdot' else S['Ws'])
    if kind == 'rowdot':
        y = (y + S['cab']).astype(np.float32)
    return P, S, (y.astype(np.float16).astype(np.float32) if tout else y), mem


def mix_launch(rs, J=17, F=5, heads=4, Cg=8, ld_extra=0, t=F32):
    mem = HostMemory()
    Ng = heads * Cg
    ld = Ng + ld_extra
    G = rs.standard_normal((F * J, ld)).astype(np.float32)
    if t:
        G = to16(G)
    ab = rs.standard_normal((F * J, 2 * heads)).astype(np.float32)
    ck = (0.1 * rs.standard_normal((heads, J, J))).astype(np.float32)
    P = record('mix', fpb=2, in_type=t, out_type=t, rows=F, K=Ng, ld=ld, J=J, heads=heads, Cg=Cg)
    P['x'], P['ab'], P['Ck'] = mem.add(G, t), mem.add(ab), mem.add(ck)
    P['out'] = mem.add(np.full((F * J, ld), 7.0), t)
    S = KA.snapshot(P, mem)
    att = emu_softmax(S['ab'], S['ck'], J, heads)
    y = emu_mix(S['G'], att, J, heads, Cg)
    out1 = S['out0'].copy()
    out1[:, :Ng] = y.astype(np.float16).astype(np.float32) if t else y
    return P, S, out1, att


# ------------------------------------------------------------------------------------------------------------------
# the restatement against a per-element loop
# ------------------------------------------------------------------------------------------------------------------
def test_expand_restatement_matches_loop():
    rs = np.random.RandomState(1)
    P, S, _, mem = expand_launch(rs, J=5, B=2, T=11, T0=4, stride=2, taps=5, Fin=2, C=12)
    y64, _ = KA.restate(P, S)
    x = mem.read(P['x'], 2 * 11 * 5 * 2).reshape(2, 11, 5, 2).astype(np.float64)
    We, be = S['We'].astype(np.float64), S['be'].astype(np.float64)
    for r in range(P['rows']):
        f, j = divmod(r, 5)
        b, t = divmod(f, 4)
        for c in range(12):
            v = be[c] + sum(We[kk * 2 + i, c] * x[b, t * 2 + kk, j, i] for kk in range(5) for i in range(2))
            assert abs(max(v, 0.0) - y64[r, c]) <= 1e-12 * (1 + abs(v))


@pytest.mark.parametrize('kind', ['rowdot', 'shrink'])
def test_dot_restatement_matches_loop(kind):
    rs = np.random.RandomState(2)
    P, S, _, mem = dot_launch(rs, kind, R=7, K=40, ld=48, heads=3)
    y64, _ = KA.restate(P, S)
    X = mem.read(P['x'], 7 * 48).reshape(7, 48).astype(np.float64)
    Wt = S['U' if kind == 'rowdot' else 'Ws'].astype(np.float64)
    for r in range(7):
        for q in range(Wt.shape[0]):
            v = sum(X[r, k] * Wt[q, k] for k in range(40)) + (S['cab'][q] if kind == 'rowdot' else 0.0)
            assert abs(v - y64[r, q]) <= 1e-12 * (1 + abs(v))


def test_mix_restatement_matches_loop():
    rs = np.random.RandomState(3)
    J, F, heads, Cg = 6, 2, 2, 4
    P, S, _, _ = mix_launch(rs, J=J, F=F, heads=heads, Cg=Cg)
    y64, _ = KA.restate(P, S)
    G, ab, ck = S['G'].astype(np.float64), S['ab'].astype(np.float64), S['ck'].astype(np.float64)
    for f in range(F):
        for h in range(heads):
            for i in range(J):
                s = [ab[f * J + i, 2 * h] + ab[f * J + j, 2 * h + 1] for j in range(J)]
                s = [v if v >= 0 else 0.2 * v for v in s]
                e = [np.exp(v - max(s)) for v in s]
                att = [e[j] / sum(e) + ck[h, i, j] for j in range(J)]
                for c in range(h * Cg, (h + 1) * Cg):
                    v = sum(att[j] * G[f * J + j, c] for j in range(J))
                    assert abs(v - y64[f * J + i, c]) <= 1e-12 * (1 + abs(v))


# ------------------------------------------------------------------------------------------------------------------
# the bounds hold for the emulation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('tin,tout', [(F32, F32), (F32, F16), (F16, F16)])
@pytest.mark.parametrize('taps', [3, 5])
def test_expand_emulation_within_bound(tin, tout, taps):
    rs = np.random.RandomState(10 + taps)
    P, S, y, _ = expand_launch(rs, taps=taps, tin=tin, tout=tout, C=1056 if taps == 5 else 96)
    assert KA.check(P, S, y)['worst'] <= 1.0


@pytest.mark.parametrize('kind,tin,tout', [(k, ti, to) for k in ('rowdot', 'shrink', 'shrink_mpjpe')
                                           for ti, to in ((F32, F32), (F16, F32), (F16, F16))
                                           if not to or k == 'shrink'])     # only a half model's shrink writes fp16
@pytest.mark.parametrize('K', [32, 160, 1600])
def test_dot_emulation_within_bound(kind, tin, tout, K):
    rs = np.random.RandomState(K)
    P, S, y, _ = dot_launch(rs, kind, K=K, tin=tin, tout=tout)
    loss = None
    if kind == 'shrink_mpjpe':
        d = (y - S['target']).astype(np.float32)
        n = np.sqrt(fma(d[:, 2], d[:, 2], fma(d[:, 1], d[:, 1], (d[:, 0] * d[:, 0]).astype(np.float32))))
        loss = float(np.float32(n.astype(np.float64).sum() / len(n)))
    rec = KA.check(P, S, y, loss)
    assert rec['worst'] <= 1.0 and (loss is None or rec['loss_worst'] <= 1.0)


@pytest.mark.parametrize('t', [F32, F16])
@pytest.mark.parametrize('J', [15, 17, 20])
def test_mix_emulation_within_bound(t, J):
    P, S, out1, _ = mix_launch(np.random.RandomState(J), J=J, t=t)
    assert KA.check(P, S, out1)['worst'] <= 1.0


def test_fp16_range_edge_is_round_to_nearest():
    """expand outputs in fp16's top binade: the emulation's inf (fp32 value >= 65520) and finite values pass; a finite
    value where the whole interval is past 65520, or inf where it is below, is refused"""
    rs = np.random.RandomState(5)
    P, S, y, _ = expand_launch(rs, tout=F16, positive=True, scale=9000.0)
    y64, e = KA.restate(P, S)
    assert np.isinf(y).any() and (np.isfinite(y) & (y > 32768)).any(), 'the data must straddle the edge'
    assert KA.check(P, S, y)['worst'] <= 1.0
    over = np.argwhere(y64 - e >= KA.F16_INF_EDGE)[0]
    bad = y.copy()
    bad[tuple(over)] = 65504.0
    with pytest.raises(GA.AuditError):
        KA.check(P, S, bad)
    under = np.argwhere(y64 + e < KA.F16_INF_EDGE)[0]
    bad = y.copy()
    bad[tuple(under)] = np.inf
    with pytest.raises(GA.AuditError):
        KA.check(P, S, bad)


def test_fp16_subnormal_outputs():
    rs = np.random.RandomState(6)
    P, S, y, _ = expand_launch(rs, tout=F16, positive=True, scale=1e-6)
    be = S['be']
    S['be'] = np.zeros_like(be)
    y = emu_expand(S['x'], S['We'], S['be']).astype(np.float16).astype(np.float32)
    assert (np.abs(y) < 2.0 ** -14).any()
    assert KA.check(P, S, y)['worst'] <= 1.0


# ------------------------------------------------------------------------------------------------------------------
# teeth
# ------------------------------------------------------------------------------------------------------------------
def _nudge(y, t, r, c, ulps):
    y = y.copy()
    if t:
        h = np.array([y[r, c]], np.float16).view(np.uint16)
        y[r, c] = (h + ulps).view(np.float16).astype(np.float32)[0]
    else:
        y[r, c] = (np.array([y[r, c]], np.float32).view(np.uint32) + ulps).view(np.float32)[0]
    return y


@pytest.mark.parametrize('kind,t', [('expand', F32), ('expand', F16), ('rowdot', F32), ('shrink', F32),
                                    ('shrink', F16)])     # the row dots are fp32 in every form
def test_moved_output_is_refused(kind, t):
    rs = np.random.RandomState(20 + t)
    if kind == 'expand':
        P, S, y, _ = expand_launch(rs, tout=t, positive=True)
    else:
        P, S, y, _ = dot_launch(rs, kind, K=256, tout=t, positive=True)
    assert KA.check(P, S, y)['worst'] <= 1.0
    y64, _ = KA.restate(P, S)
    assert (y64 > 0).all()                       # operands of one sign: S = |y|
    r, c = 3, 1
    with pytest.raises(GA.AuditError):
        KA.check(P, S, _nudge(y, t, r, c, 2 if t else 16))


@pytest.mark.parametrize('kind', ['expand', 'shrink'])
def test_row_of_the_neighbouring_frame_is_refused(kind):
    rs = np.random.RandomState(30)
    if kind == 'expand':
        P, S, y, _ = expand_launch(rs)
        S2 = dict(S, x=S['x'].copy())
        S2['x'][4] = S['x'][4 + P['J']]          # output row 4 read frame t + 1
        y = emu_expand(S2['x'], S['We'], S['be'])
    else:
        P, S, y, _ = dot_launch(rs, kind, R=40)
        P['J'] = 17
        X = S['X'].copy()
        X[5] = X[5 + 17]
        y = lane_dot(X, S['Ws'])
    with pytest.raises(GA.AuditError):
        KA.check(P, S, y)


def test_mix_with_the_next_heads_attention_is_refused():
    rs = np.random.RandomState(40)
    P, S, out1, att = mix_launch(rs, heads=4)
    assert KA.check(P, S, out1)['worst'] <= 1.0
    out2 = out1.copy()
    out2[:, :P['K']] = emu_mix(S['G'], att, P['J'], 4, P['Cg'], head_of=lambda h: h + 1 if h == 1 else h)
    with pytest.raises(GA.AuditError):
        KA.check(P, S, out2)


def test_write_past_the_owned_columns_is_refused():
    rs = np.random.RandomState(50)
    P, S, out1, _ = mix_launch(rs, ld_extra=8)
    assert KA.check(P, S, out1)['worst'] <= 1.0
    out2 = out1.copy()
    out2[3, P['K']] = 0.5
    with pytest.raises(GA.AuditError):
        KA.check(P, S, out2)


def test_moved_loss_is_refused():
    rs = np.random.RandomState(60)
    P, S, y, _ = dot_launch(rs, 'shrink_mpjpe', R=30)
    l64, _ = KA.mpjpe_loss(y, S['target'])
    assert KA.check(P, S, y, float(np.float32(l64)))['loss_worst'] <= 1.0
    moved = float((np.array([l64], np.float32).view(np.uint32) + 16).view(np.float32)[0])
    with pytest.raises(GA.AuditError):
        KA.check(P, S, y, moved)


def test_reads_stay_inside_the_allocations():
    """the snapshot of a strided expand, a row-dot over ld > K and a mix reads only inside their buffers (HostMemory
    asserts), and the tags name the variant and the types"""
    rs = np.random.RandomState(70)
    P, S, y, _ = expand_launch(rs, taps=5, T=15, T0=3, stride=5, tin=F16, tout=F16)
    assert 'expand:kft10:f16->f16' in KA.check(P, S, y)['tags']
    P, S, y, _ = dot_launch(rs, 'rowdot', K=64, ld=96, heads=1)
    assert 'rowdot:rowdot<2>:f32->f32' in KA.check(P, S, y)['tags']


# ------------------------------------------------------------------------------------------------------------------
# the derived constants
# ------------------------------------------------------------------------------------------------------------------
def _bn_params(rs, n, p):
    return {p + 'weight': (1 + 0.2 * rs.standard_normal(n)).astype(np.float32),
            p + 'bias': (0.3 * rs.standard_normal(n)).astype(np.float32),
            p + 'running_mean': (0.3 * rs.standard_normal(n)).astype(np.float32),
            p + 'running_var': (0.5 + rs.random_sample(n)).astype(np.float32)}


def test_fold_bounds_hold_for_the_fp32_fold_and_refuse_a_swapped_tap():
    rs = np.random.RandomState(80)
    C, Fin, taps = 32, 2, 3
    sd = {'expand_conv.weight': (0.5 * rs.standard_normal((C, Fin, taps, 1))).astype(np.float32)}
    sd.update(_bn_params(rs, Fin, 'init_bn.'))
    sd.update(_bn_params(rs, C, 'expand_bn.'))
    f = np.float32

    def bn(p, n):
        s = (sd[p + 'weight'] / np.sqrt(sd[p + 'running_var'] + f(1e-5))).astype(f)
        return s, (sd[p + 'bias'] - sd[p + 'running_mean'] * s).astype(f)
    si, ti = bn('init_bn.', Fin)
    se, te = bn('expand_bn.', C)
    w = sd['expand_conv.weight'].reshape(C, Fin, taps)
    We = np.zeros((taps * Fin, C), f)
    acc = np.zeros(C, f)
    for kk in range(taps):
        for i in range(Fin):
            We[kk * Fin + i] = (w[:, i, kk] * si[i]).astype(f) * se
            acc = fma(w[:, i, kk], ti[i], acc)
    be = (se * acc + te).astype(f)
    We64, eWe, be64, ebe = KA.fold_bounds(sd, taps, Fin)
    assert KA.within(We, We64, eWe, 'We') <= 1.0 and KA.within(be, be64, ebe, 'be') <= 1.0
    with pytest.raises(GA.AuditError):
        KA.within(We[[2, 3, 0, 1, 4, 5]], We64, eWe, 'We')


def test_collapse_bounds_hold_for_the_fp32_collapse():
    rs = np.random.RandomState(90)
    Ci, C = 24, 40
    tw, pw = (rs.standard_normal((2, Ci, C, 1)) / 5).astype(np.float32)
    tb, pb = (rs.standard_normal((2, Ci)) / 5).astype(np.float32)
    wc = rs.standard_normal(2 * Ci).astype(np.float32)
    U64, eU, cab64, ecab = KA.collapse_bounds(tw, tb, pw, pb, wc)
    Uf = np.stack([(wc[:Ci, None] * tw[..., 0]).sum(0), (wc[Ci:, None] * pw[..., 0]).sum(0)]).astype(np.float32)
    cab = np.array([(wc[:Ci] * tb).sum(), (wc[Ci:] * pb).sum()], np.float32)
    assert KA.within(Uf, U64, eU, 'U') <= 1.0 and KA.within(cab, cab64, ecab, 'cab') <= 1.0
    with pytest.raises(GA.AuditError):
        KA.within(Uf[::-1], U64, eU, 'U')
