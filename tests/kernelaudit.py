"""Per-launch audit of the kernels of the forward other than the GEMMs: every expand, theta/phi row-dot, attention-mix
and shrink launch (csrc/gast_api.cu launch_expand, launch_rowdot, run_global, launch_shrink) held to fp64 of its own
operands.

Test infrastructure, the companion of tests/gemmaudit.py.  gast_debug_set_kernel_audit calls back just before and
just after each of these launches with a gast_kernel_audit record (include/gast_b200.h), the stream synchronised.
`Auditor` snapshots, before the launch, the addresses the launch reads (every span from the first to the last element
the kernel reads, so inside one allocation) and its output window; after it, the output window again.  `check`
restates the launch in fp64 from the record and holds every element to a bound derived from the kernel's fp32
arithmetic (u = 2^-24, S = sum |a w| of the element over its products, exact on the stored operands):

  expand:  out[r, c] = relu(be[c] + sum_k We[k, c] x_r[k]), k over the taps and features (KF = taps Fin), x_r[k] =
           x[((b T + t stride + kk) J + j) Fin + i] for r = (b T0 + t) J + j.  The kernel runs one chain of KF FMAs
           that starts from be: (KF + 1) u (|be| + S).
  rowdot:  ab[r, q] = X[r] . U[q] + cab[q].  Each lane chains 4 ceil(K / 128) FMAs, then a 5-step butterfly (the
           shuffle sum, or rowdot8's halving butterfly), then the cab add: (4 ceil(K / 128) + 6) u (S + |cab|).
           The output is fp32 in every form.
  mix:     Y[f J + i, n] = sum_j att_{n / Cg}[f, i, j] G[f J + j, n], restated from the stored G, the ab the row-dot
           launch before it wrote, and Ck, with gemmaudit's softmax and J-term chain bound (GA.attention, GA._global)
           at e_G = 0.
  shrink:  y[r, o] = X[r] . Ws[o]: (4 ceil(K / 128) + 5) u S.
  shrink_mpjpe:  y as shrink; the loss against fp64 of mean_r ||y_dev[r] - target[r]|| from the device's own y: each
           term takes the difference, two FMAs and a square root in fp32 (< 4 u relative), the sum is double and the
           result one float rounding: |loss - loss64| <= 5 u loss64 + 2^-149.

fp16 outputs (the expand and mix at either fp16 form, the shrink of a half model) round the fp32 result once more:
the bound adds 2^-11 (|y64| + e) + 2^-25.  Past fp16's range round to nearest is IEEE's: an element whose whole
interval [y64 - e, y64 + e] is at or above 65520 in magnitude must be inf of its sign, one whose interval is below
65520 must be finite, and either is accepted in between.  fp16 inputs are read as stored and widened exactly.
Columns [width, ld) of an output window that the launch does not own must be bitwise what they were before it (the
mix's Y when ld > heads Cg).

`fold_bounds` and `collapse_bounds` hold the derived constants the launches read to fp64 of the module parameters:
We / be of expand_fold_kernel (both BatchNorms folded into the expand conv) and U / cab of global_collapse_kernel
(theta and phi collapsed through concat_project), so that a bug in preparing them is caught, not restated.
"""
import numpy as np

import gemmaudit as GA

U = GA.U
F16_HALF_ULP = 2.0 ** -11
F16_SUB = 2.0 ** -25
F16_INF_EDGE = 65520.0          # the smallest magnitude round-to-nearest fp16 takes to inf
KINDS = ('expand', 'rowdot', 'mix', 'shrink', 'shrink_mpjpe')
TYPES = ('f32', 'f16')
BN_EPS = 1e-5

FIELDS = ('index', 'gemm_index', 'kind', 'variant', 'fpb', 'block', 'in_type', 'out_type', 'rows', 'K', 'ld', 'J',
          'T', 'T0', 'stride', 'taps', 'Fin', 'heads', 'Cg')
POINTERS = ('x', 'We', 'be', 'U', 'cab', 'ab', 'Ck', 'Ws', 'target', 'loss', 'out')


def params(d):
    """plain dict of a gast_kernel_audit record (ctypes)"""
    P = {k: int(getattr(d, k)) for k in FIELDS}
    for k in POINTERS:
        P[k] = getattr(d, k) or 0
    return P


def _read(mem, ptr, n, t):
    return mem.read16(ptr, n) if t else mem.read(ptr, n)


def _span(mem, ptr, offs, t):
    """elements at offsets offs (any shape) from ptr, from one span read"""
    offs = np.asarray(offs, np.int64)
    lo, hi = int(offs.min()), int(offs.max()) + 1
    return _read(mem, ptr + (2 if t else 4) * lo, hi - lo, t)[offs - lo]


def nq(P):
    return 2 * P['heads']


def window(P):
    """(rows, ld, width, type) of the launch's output window: ld floats per row, the first width owned"""
    k = KINDS[P['kind']]
    if k == 'expand':
        return P['rows'], P['ld'], P['K'], P['out_type']
    if k == 'rowdot':
        return P['rows'], nq(P), nq(P), 0
    if k == 'mix':
        return P['rows'] * P['J'], P['ld'], P['K'], P['out_type']
    return P['rows'], 3, 3, P['out_type']


def expand_offsets(P):
    """(rows, KF) offsets into x of each output row's taps and features"""
    r = np.arange(P['rows'])
    f, j = r // P['J'], r % P['J']
    b, t = f // P['T0'], f % P['T0']
    kk = np.repeat(np.arange(P['taps']), P['Fin'])
    i = np.tile(np.arange(P['Fin']), P['taps'])
    return (((b * P['T'] + t * P['stride'])[:, None] + kk[None, :]) * P['J'] + j[:, None]) * P['Fin'] + i[None, :]


def _rows(mem, ptr, R, ld, w, t):
    return _span(mem, ptr, np.arange(R)[:, None] * ld + np.arange(w)[None, :], t)


def snapshot(P, mem):
    """the launch's operands and its output window, read before it runs"""
    k = KINDS[P['kind']]
    S = {}
    if k == 'expand':
        KF = P['taps'] * P['Fin']
        S['x'] = _span(mem, P['x'], expand_offsets(P), P['in_type'])
        S['We'] = mem.read(P['We'], KF * P['K']).reshape(KF, P['K'])
        S['be'] = mem.read(P['be'], P['K'])
    elif k == 'rowdot':
        S['X'] = _rows(mem, P['x'], P['rows'], P['ld'], P['K'], P['in_type'])
        S['U'] = mem.read(P['U'], nq(P) * P['K']).reshape(nq(P), P['K'])
        S['cab'] = mem.read(P['cab'], nq(P))
    elif k == 'mix':
        R = P['rows'] * P['J']
        S['G'] = _rows(mem, P['x'], R, P['ld'], P['K'], P['in_type'])
        S['ab'] = mem.read(P['ab'], R * nq(P)).reshape(R, nq(P))
        S['ck'] = mem.read(P['Ck'], P['heads'] * P['J'] ** 2).reshape(P['heads'], P['J'], P['J'])
    else:
        S['X'] = _rows(mem, P['x'], P['rows'], P['ld'], P['K'], P['in_type'])
        S['Ws'] = mem.read(P['Ws'], 3 * P['K']).reshape(3, P['K'])
        if k == 'shrink_mpjpe':
            S['target'] = mem.read(P['target'], 3 * P['rows']).reshape(P['rows'], 3)
    S['out0'] = read_out(P, mem)
    return S


def read_out(P, mem):
    """the output window up to the last element the launch writes, NaN-padded to full rows"""
    R, ld, w, t = window(P)
    n = (R - 1) * ld + w
    win = np.full(R * ld, np.nan, np.float32)
    win[:n] = _read(mem, P['out'] if KINDS[P['kind']] != 'rowdot' else P['ab'], n, t)
    return win.reshape(R, ld)


# ----------------------------------------------------------------------------------------------------------------
# fp64 restatement and bounds
# ----------------------------------------------------------------------------------------------------------------
def chain(K):
    """FMAs in one lane's chain of a warp-per-row dot product over K"""
    return 4 * -(-K // 128)


def restate(P, S):
    """(y64, e): the launch's owned output in fp64 and the elementwise bound of its fp32 arithmetic (before the
    rounding of an fp16 output)"""
    k = KINDS[P['kind']]
    if k == 'expand':
        x, We, be = S['x'].astype(np.float64), S['We'].astype(np.float64), S['be'].astype(np.float64)
        y = np.maximum(be + x @ We, 0.0)
        KF = P['taps'] * P['Fin']
        return y, (KF + 1) * U * (np.abs(be) + np.abs(x) @ np.abs(We))
    if k == 'rowdot':
        X, Uq, cab = S['X'].astype(np.float64), S['U'].astype(np.float64), S['cab'].astype(np.float64)
        return X @ Uq.T + cab, (chain(P['K']) + 6) * U * (np.abs(X) @ np.abs(Uq).T + np.abs(cab))
    if k == 'mix':
        P2 = dict(F=P['rows'], J=P['J'], N=P['K'], heads=P['heads'], Cg=P['Cg'])
        G = S['G'].astype(np.float64)
        return GA._global(P2, dict(ab=S['ab'], ck=S['ck']), G, np.zeros_like(G), 0.0)
    X, Ws = S['X'].astype(np.float64), S['Ws'].astype(np.float64)
    return X @ Ws.T, (chain(P['K']) + 5) * U * (np.abs(X) @ np.abs(Ws).T)


def mpjpe_loss(y, target):
    """(loss64, bound): fp64 of mean ||y - target|| from the device's y, and the bound of the kernel's loss"""
    l64 = float(np.mean(np.sqrt(((y.astype(np.float64) - target.astype(np.float64)) ** 2).sum(axis=1))))
    return l64, 5 * U * l64 + 2.0 ** -149


class AuditError(GA.AuditError):
    pass


def name(P):
    return 'kernel launch %d (%s, variant %d, fpb %d, %s -> %s, rows %d K %d ld %d J %d)' % (
        P['index'], KINDS[P['kind']], P['variant'], P['fpb'], TYPES[P['in_type']], TYPES[window(P)[3]], P['rows'],
        P['K'], P['ld'], P['J'])


def check(P, S, out1, loss=None):
    """hold a launch's output window (read after it ran; loss: the shrink_mpjpe loss it wrote) to the fp64
    restatement; -> its record.  Raises AuditError naming the launch and the worst element."""
    R, ld, w, t = window(P)
    y = out1[:, :w].astype(np.float64)
    y64, e = restate(P, S)
    if t:
        tot = e + F16_HALF_ULP * (np.abs(y64) + e) + F16_SUB
        must_inf = (y64 - e >= F16_INF_EDGE) | (y64 + e <= -F16_INF_EDGE)
        may_inf = np.where(y >= 0, y64 + e >= F16_INF_EDGE, y64 - e <= -F16_INF_EDGE)
        inf = np.isinf(y)
        err = np.where(inf, 0.0, np.abs(y - y64))
        bad = np.where(inf, ~may_inf, must_inf | np.isnan(y))
    else:
        tot = e
        err = np.abs(y - y64)
        bad = ~np.isfinite(y)
    ratio = np.where(tot > 0, err / np.where(tot > 0, tot, 1.0), np.where(err > 0, np.inf, 0.0))
    ratio[bad] = np.inf
    worst = float(ratio.max()) if ratio.size else 0.0
    if worst > 1.0:
        r, c = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        raise AuditError('%s: element (%d, %d) = %r, fp64 %r, |err| %.3e > bound %.3e (%d elements past it)' % (
            name(P), r, c, float(y[r, c]), float(y64[r, c]), err[r, c], tot[r, c], int((ratio > 1).sum())))
    tail0, tail1 = S['out0'][:-1, w:], out1[:-1, w:]
    if tail0.size and not np.array_equal(tail0.view(np.uint32), tail1.view(np.uint32)):
        r, c = np.argwhere(tail0.view(np.uint32) != tail1.view(np.uint32))[0]
        raise AuditError('%s: wrote column %d of row %d, past its %d columns (%r -> %r)' % (
            name(P), w + c, r, w, float(tail0[r, c]), float(tail1[r, c])))
    rec = dict(index=P['index'], gemm_index=P['gemm_index'], kind=KINDS[P['kind']], variant=P['variant'],
               fpb=P['fpb'], block=P['block'], types=(TYPES[P['in_type']], TYPES[t]), rows=P['rows'], K=P['K'],
               J=P['J'], worst=worst, loss_worst=None, tags=tags(P))
    if loss is not None:
        l64, lb = mpjpe_loss(out1[:, :3], S['target'])
        rec['loss_worst'] = abs(loss - l64) / lb
        if not rec['loss_worst'] <= 1.0:
            raise AuditError('%s: loss %r, fp64 of the device y %r, |err| %.3e > bound %.3e' % (
                name(P), loss, l64, abs(loss - l64), lb))
    return rec


def variant_tag(P):
    k = KINDS[P['kind']]
    if k == 'expand':
        return 'kft%d' % P['variant']
    if k == 'rowdot':
        return 'rowdot8' if P['variant'] == 0 else 'rowdot<%d>' % P['variant']
    return k


def tags(P):
    """kind x variant x (in, out) type, and the edges of the launch, for the coverage count"""
    R, ld, w, t = window(P)
    out = {'%s:%s:%s->%s' % (KINDS[P['kind']], variant_tag(P), TYPES[P['in_type']], TYPES[t])}
    k = KINDS[P['kind']]
    if k == 'expand':
        if P['K'] > 1024:
            out.add('expand:two_chunks:' + TYPES[t])
        if 256 % (min(P['K'], 1024) // 4):
            out.add('expand:surplus_threads')
        if P['rows'] % 128:
            out.add('expand:partial_block')
        if P['T0'] == 1 and P['T'] == P['taps']:
            out.add('expand:one_window')
        elif P['T0'] > 1 and P['stride'] == 1 and P['T'] == P['taps'] - 1 + P['T0']:
            out.add('expand:stride1_windows')
    if k == 'rowdot' and P['variant'] == 0 and P['rows'] % 16:
        out.add('rowdot8:odd_warp_rows')
    if k == 'rowdot' and P['variant'] == 8 and P['in_type']:
        out.add('rowdot<8>:f16')
    if k == 'mix':
        out.add('mix:J%d' % P['J'])
        if P['fpb'] == 1:
            out.add('mix:fpb1')
        elif P['rows'] % P['fpb']:
            out.add('mix:partial_block')
    if k == 'shrink_mpjpe':
        out.add('shrink_mpjpe:one_block' if P['rows'] <= 8 else
                'shrink_mpjpe:grid_stride' if P['rows'] > 8 * 1024 else 'shrink_mpjpe:blocks')
    return out


# ----------------------------------------------------------------------------------------------------------------
# the derived constants against the module parameters
# ----------------------------------------------------------------------------------------------------------------
def _bn(sd, p, n):
    g = sd[p + 'weight'].astype(np.float64)
    s = g / np.sqrt(sd[p + 'running_var'].astype(np.float64) + BN_EPS)
    return s, sd[p + 'bias'].astype(np.float64) - sd[p + 'running_mean'].astype(np.float64) * s


def fold_bounds(sd, taps, Fin):
    """(We64, eWe, be64, ebe): expand_fold_kernel's We (taps Fin, C) and be (C) in fp64 from the state dict `sd`
    (numpy) and their bounds: each BatchNorm scale is a few fp32 roundings (the variance add, sqrt, divide), We two
    products more; be chains taps Fin FMAs into se acc + te."""
    w = sd['expand_conv.weight'].astype(np.float64).reshape(-1, Fin, taps)      # (C, Fin, taps)
    C = w.shape[0]
    si, ti = _bn(sd, 'init_bn.', Fin)
    se, te = _bn(sd, 'expand_bn.', C)
    Wk = w.transpose(2, 1, 0).reshape(taps * Fin, C)                          # [kk Fin + i][c]
    sik = np.tile(si, taps)[:, None]
    tik = np.tile(ti, taps)[:, None]
    We64 = Wk * sik * se[None, :]
    eWe = 12 * U * np.abs(We64)
    acc = (Wk * tik).sum(axis=0)
    mag = (np.abs(Wk) * np.abs(tik)).sum(axis=0)
    rm_i = np.tile(np.abs(sd['init_bn.running_mean'].astype(np.float64)) * si, taps)[:, None]
    eti = 8 * U * (np.tile(np.abs(sd['init_bn.bias'].astype(np.float64)), taps)[:, None] + rm_i)
    rm_e = np.abs(sd['expand_bn.running_mean'].astype(np.float64)) * np.abs(se)
    be64 = se * acc + te
    ebe = ((taps * Fin + 8) * U * (np.abs(se) * mag + np.abs(sd['expand_bn.bias'].astype(np.float64)) + rm_e)
           + np.abs(se) * (np.abs(Wk) * eti).sum(axis=0))
    return We64, eWe, be64, ebe


def collapse_bounds(tw, tb, pw, pb, wc):
    """(U64, eU, cab64, ecab) of one head: U[2h] = wc[:Ci] theta_w, U[2h + 1] = wc[Ci:] phi_w, cab likewise from the
    biases, and their bounds (8 strided chains of Ci / 8 FMAs summed in fp32, or one chain of Ci for cab)"""
    Ci = tw.shape[0]
    wa, wb = wc[:Ci].astype(np.float64), wc[Ci:].astype(np.float64)
    tw, pw = tw.reshape(Ci, -1).astype(np.float64), pw.reshape(Ci, -1).astype(np.float64)
    tb, pb = tb.astype(np.float64), pb.astype(np.float64)
    U64 = np.stack([wa @ tw, wb @ pw])
    eU = (-(-Ci // 8) + 8) * U * np.stack([np.abs(wa) @ np.abs(tw), np.abs(wb) @ np.abs(pw)])
    cab64 = np.array([wa @ tb, wb @ pb])
    ecab = Ci * U * np.array([np.abs(wa) @ np.abs(tb), np.abs(wb) @ np.abs(pb)])
    return U64, eU, cab64, ecab


def within(dev, ref, bound, what):
    err = np.abs(np.asarray(dev, np.float64) - ref)
    ratio = float((err / np.where(bound > 0, bound, 1e-300)).max()) if err.size else 0.0
    if not ratio <= 1.0:
        i = np.unravel_index(int(np.argmax(err / np.where(bound > 0, bound, 1e-300))), err.shape)
        raise AuditError('%s: element %s = %r, fp64 %r, bound %.3e' % (what, i, float(np.asarray(dev)[i]),
                                                                       float(ref[i]), float(bound[i])))
    return ratio


# ----------------------------------------------------------------------------------------------------------------
# the hook
# ----------------------------------------------------------------------------------------------------------------
class Auditor(object):
    """the callback of gast_debug_set_kernel_audit: snapshots each launch, checks it after it ran and keeps the
    records (self.records), the raw parameters and snapshots when keep is set (self.launches), and the first failure
    (self.failure, also returned to the library so that the call fails).  kinds: the kinds to audit (others pass)."""

    def __init__(self, mem=None, kinds=KINDS, keep=False):
        from gast_b200 import _lib
        import gemmaudit_half as GAH
        self.mem = mem or GAH.DeviceMemory()
        self.kinds = set(kinds)
        self.keep = keep
        self.records = []
        self.launches = []
        self.failure = None
        self._pending = {}
        self.fn = _lib.KernelAuditFn(self._call)

    def _call(self, phase, d, user):
        try:
            P = params(d.contents)
            if KINDS[P['kind']] not in self.kinds:
                return 0
            if phase == 0:
                self._pending[P['index']] = (P, snapshot(P, self.mem))
            else:
                P0, S = self._pending.pop(P['index'])
                out1 = read_out(P0, self.mem)
                loss = float(self.mem.read(P0['loss'], 1)[0]) if KINDS[P0['kind']] == 'shrink_mpjpe' else None
                self.records.append(check(P0, S, out1, loss))
                if self.keep:
                    self.launches.append((P0, S, out1))
            return 0
        except Exception as ex:   # the library fails the call; the message is kept for the test
            if self.failure is None:
                import traceback
                self.failure = '%s: %s\n%s' % (type(ex).__name__, ex, traceback.format_exc(limit=-4))
            return 1

    def install(self, lib, h):
        rc = lib.gast_debug_set_kernel_audit(h, self.fn, None)
        assert rc == 0


def report_line(rec):
    return '%6d %-12s %-10s %s->%s rows %7d K %5d J %2d fpb %3d worst %.3e loss %s\n' % (
        rec['index'], rec['kind'], variant_tag_rec(rec), rec['types'][0], rec['types'][1], rec['rows'], rec['K'],
        rec['J'], rec['fpb'], rec['worst'], '-' if rec['loss_worst'] is None else '%.3e' % rec['loss_worst'])


def variant_tag_rec(rec):
    return variant_tag(dict(kind=KINDS.index(rec['kind']), variant=rec['variant']))
