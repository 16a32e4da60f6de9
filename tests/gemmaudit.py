"""Per-launch audit of the GEMMs: each launch of launch_gemm (csrc/gast_api.cu) held to fp64 of its own fp32 operands.

Test infrastructure.  gast_debug_set_gemm_audit calls back just before and just after every GEMM launch of a handle
with a gast_gemm_audit record (include/gast_b200.h), the stream synchronised.  `Auditor` snapshots, before the launch,
exactly the addresses the launch reads -- every A segment's rows under its frame map and taps, W, bias, the residual
rows under res_map, the SemCH and global-attention operands -- and the output window; after it, the output window
again.  Every read is the span from the first to the last address the kernel itself reads (the output window ends at
the last element the kernel writes), so it stays inside one allocation.  `check` then restates the launch in fp64 from
the GemmP contract (csrc/gast_common.cuh, gemm_epilogue in csrc/gemm_ffma.cuh):

  A[f J + j, kcol(s) + tap Kc + c] = base_s[(map_s(f) J + j) ld_s + tap tap_stride_s + c],   H = A W^T
  plain:  relu?(H + bias) + res[(map_res(f) J + j) res_ld]
  SemCH:  column tile t of mask m = t / tiles_per_mask holds 64 self (W0) and 64 neighbour (W1) products; output
          column m C + c (c = 64 (t % tiles_per_mask) + c' < C) is relu?(shift[m C + c] + sum_z coef_m[z C + c] H_z),
          z over joint i's neighbours nbr_m, H_z the self column of row i when the neighbour is i itself and the
          neighbour column of the neighbour's row otherwise
  global: G = H + bg; att_h[i, j] = softmax_j(LeakyReLU_0.2(ab[i, 2h] + ab[j, 2h + 1])) + ck[h, i, j];
          y[i, n] = sum_j att_{n / Cg}[i, j] G[j, n]

and holds every element to a bound derived from the arithmetic of the core and form that ran (u = 2^-24, S = sum_k
|a_k w_k| of the element's row and column, all in exact arithmetic on the fp32 operands):

  FFMA core: one fused multiply-add chain over K, |H^ - H| <= K u S.
  3xTF32 and F16X3: x = x_hi + x_lo + d_x with x_hi, x_lo of 11 significant bits each, |x_lo| <= 2^-11 |x| and
      |d_x| <= 2^-22 |x|; the product drops x_lo y_lo and the d terms: <= 3 2^-22 |a w|.  The tensor core aligns the
      addends of each MMA (k products and the accumulator) to the largest and truncates them, each by less than one
      fp32 ulp of that largest addend: <= (k + 1) 2^-23 of the MMA's absolute sum, and a 16-K partial takes 6 k8 MMAs
      (3xTF32) or 3 k16 MMAs (F16X3), each with the partial's absolute sum bounding its own.  Each partial is then
      added into the fp32 tile sum with one round-to-nearest: <= u sum_{so far}, over K / 16 partials.
      tau = 3 2^-22 + n_mma (k + 1) 2^-23 + (K / 16) u.
      F16X3 also scales A per row and 32-K stage (its max m to [2^14, 2^15)) and W per matrix, and rounds in fp16,
      whose subnormals are 2^-24 apart: an absolute 2^-24 per operand in scaled units, 2^-38 m (A) and 2^-38 max|W|
      unscaled, so it adds 2^-38 (sum_k m_k |w_k| + max|W| sum_k |a_k|).
  1xTF32: x = x_hi + d_x with |d_x| <= 2^-11 |x|: <= (2^-10 + 2^-22) |a w| per product, 2 k8 MMAs per partial.
  Every form adds u for the bias add (one rounding of H + bias, |H + bias| <= S + |bias|).

  plain:   |y - y64| <= tau (S + |bias|) + 2^-23 (|y64| + |res|)        (ReLU is 1-Lipschitz; the residual add rounds
                                                                         once, with slack for the bound on its input)
  SemCH:   the bound e_z on each H_z carried through the mix, sum_z |coef_z| e_z, plus the mix's own chain of
           n + 1 roundings (n neighbours and the shift): (n + 1) u (|shift| + sum_z |coef_z| (|H_z| + e_z))
  global:  e_G = tau (S + |bg|) carried through the attention, sum_j |att_j| e_Gj, plus the fp32 softmax's error on
           att (the score add and LeakyReLU 2^-23 |s|, the shift by the row max 2 u smax, expf 2 ulp, the J-term
           sum, the reciprocal and the C_k add: eps = 2 (6 smax u + 2^-22) + (J + 2) u relative to the softmax,
           plus u |att|), times |G_j|, plus the J-term chain of the mix, J u sum_j |att_j| (|G_j| + e_Gj).

A second check holds the tensor-core launches to the numpy emulations of their form (tests/f16x3ref.py gemm and
gemm_3xtf32, tests/tf32ref.py tf32) on the dense gathered A, through the same epilogue, at a relative L2 bar, as
tests/test_gpu_tc_act_tma.py does for the dense debug GEMM.  Columns [width, ld_out) of the output window that the
launch does not own must be bitwise what they were before it.
"""
import os

import numpy as np

import f16x3ref as F16
import tf32ref as TF

U = 2.0 ** -24
EPI_NAMES = ('plain', 'semch', 'global')
FORMS = {-1: 'ffma', 0: '3xtf32', 1: 'tf32', 2: 'f16x3'}
EMU_L2_BAR = 2e-6
EMU_MAX_ROWS = 2048


# ----------------------------------------------------------------------------------------------------------------
# the launch's parameters and operands
# ----------------------------------------------------------------------------------------------------------------
def params(d):
    """plain dict of a gast_gemm_audit record (ctypes)"""
    P = {k: int(getattr(d, k)) for k in ('index', 'epi', 'core', 'tc_form', 'tma_mask', 'nseg', 'ldw', 'N', 'F', 'J',
                                          'fpt', 'ld_out', 'relu', 'res_ld', 'C', 'tiles_per_mask', 'heads', 'Cg')}
    P['segs'] = [dict(base=d.seg[s].base or 0, ld=d.seg[s].ld, K=d.seg[s].K, Kc=d.seg[s].Kc,
                      tap_stride=int(d.seg[s].tap_stride),
                      map=(d.seg[s].T_out, d.seg[s].T_in, d.seg[s].t_mul, d.seg[s].t_off)) for s in range(P['nseg'])]
    for k in ('W', 'out', 'bias', 'res', 'shift', 'ab', 'ck', 'bg'):
        P[k] = getattr(d, k) or 0
    P['coef'] = [d.coef[0] or 0, d.coef[1] or 0]
    P['res_map'] = (d.res_T_out, d.res_T_in, d.res_t_mul, d.res_t_off)
    P['nbr'] = [(list(d.nbr_row_ptr[m]), list(d.nbr_col[m])) for m in range(2)]
    return P


def map_frames(m, f):
    T_out, T_in, t_mul, t_off = m
    f = np.asarray(f, np.int64)
    return (f // T_out) * T_in + (f % T_out) * t_mul + t_off


def nmasks(P):
    return P['N'] // (128 * P['tiles_per_mask']) if P['epi'] == 1 else 0


def width(P):
    """output columns the launch owns: N, or for SemCH the masks' C channels each"""
    return nmasks(P) * P['C'] if P['epi'] == 1 else P['N']


def nnz(P, m):
    return P['nbr'][m][0][P['J']]


class DeviceMemory(object):
    """reads fp32 spans of device memory at raw addresses (the stream is synchronised by the library)"""

    def read(self, ptr, n):
        import torch

        class _Span(object):
            __cuda_array_interface__ = {'shape': (int(n),), 'typestr': '<f4', 'data': (int(ptr), False),
                                        'version': 2, 'strides': None}
        return torch.as_tensor(_Span(), device='cuda').cpu().numpy().copy()


def _rows(mem, base, offs, w):
    """rows of w floats at float offsets offs (any shape) from base, from one span read -> offs.shape + (w,)"""
    offs = np.asarray(offs, np.int64)
    lo, hi = int(offs.min()), int(offs.max()) + w
    buf = mem.read(base + 4 * lo, hi - lo)
    return buf[(offs - lo)[..., None] + np.arange(w)]


def gather_a(P, mem):
    """the dense A (F J, K) of the launch, segment by segment"""
    F, J = P['F'], P['J']
    f = np.repeat(np.arange(F), J)
    j = np.tile(np.arange(J), F)
    parts = []
    for s in P['segs']:
        taps = s['K'] // s['Kc']
        src = map_frames(s['map'], f) * J + j
        offs = src[:, None] * s['ld'] + np.arange(taps)[None, :] * s['tap_stride']
        parts.append(_rows(mem, s['base'], offs, s['Kc']).reshape(F * J, s['K']))
    return np.concatenate(parts, axis=1)


def snapshot(P, mem):
    """the launch's operands and its output window, read before it runs"""
    F, J, N, K = P['F'], P['J'], P['N'], P['ldw']
    R = F * J
    S = {'A': gather_a(P, mem), 'W': mem.read(P['W'], N * K).reshape(N, K)}
    if P['bias']:
        S['bias'] = mem.read(P['bias'], N)
    if P['epi'] == 0 and P['res']:
        src = map_frames(P['res_map'], np.repeat(np.arange(F), J)) * J + np.tile(np.arange(J), F)
        S['res'] = _rows(mem, P['res'], src * P['res_ld'], N)
    if P['epi'] == 1:
        nm = nmasks(P)
        S['coef'] = [mem.read(P['coef'][m], nnz(P, m) * P['C']).reshape(-1, P['C']) for m in range(nm)]
        if P['shift']:
            S['shift'] = mem.read(P['shift'], nm * P['C'])
    if P['epi'] == 2:
        S['ab'] = mem.read(P['ab'], R * 2 * P['heads']).reshape(R, 2 * P['heads'])
        S['ck'] = mem.read(P['ck'], P['heads'] * J * J).reshape(P['heads'], J, J)
        if P['bg']:
            S['bg'] = mem.read(P['bg'], N)
    S['out0'] = read_out(P, mem)
    return S


def read_out(P, mem):
    """the output window [0, F J) x [0, ld_out), up to the last element the launch writes, NaN-padded to full rows"""
    R, ld = P['F'] * P['J'], P['ld_out']
    n = (R - 1) * ld + width(P)
    win = np.full(R * ld, np.nan, np.float32)
    win[:n] = mem.read(P['out'], n)
    return win.reshape(R, ld)


# ----------------------------------------------------------------------------------------------------------------
# fp64 restatement and bounds
# ----------------------------------------------------------------------------------------------------------------
def tau(form, K):
    """relative bound of one GEMM output on sum |a w| (module docstring)"""
    if form == -1:
        return K * U + U
    acc = (K / 16.0) * U + U
    if form == 0:
        return 3 * 2.0 ** -22 + 6 * 9 * 2.0 ** -23 + acc
    if form == 2:
        return 3 * 2.0 ** -22 + 3 * 17 * 2.0 ** -23 + acc
    return 2.0 ** -10 + 2.0 ** -22 + 2 * 9 * 2.0 ** -23 + acc


def gemm_bound(P, S, form):
    """(H64, e_H): the exact product and the bound on the device's product, both (F J, N) fp64"""
    A, W = S['A'].astype(np.float64), S['W'].astype(np.float64)
    H = A @ W.T
    aA, aW = np.abs(A), np.abs(W)
    e = tau(form, A.shape[1]) * (aA @ aW.T)
    if form == 2:
        R, K = A.shape
        m = np.repeat(np.abs(A).reshape(R, K // 32, 32).max(axis=2), 32, axis=1)
        e += 2.0 ** -38 * (m @ aW.T + aA.sum(axis=1, keepdims=True) * aW.max(initial=0.0))
    return H, e


def restate(P, S, form=None, H=None):
    """(y64, bound): the launch's output columns [0, width) in fp64 and the elementwise bound for `form` (default the
    form that ran).  H: a stand-in product (the emulation), whose epilogue is then restated the same way."""
    form = P['tc_form'] if form is None else form
    Hx, e = gemm_bound(P, S, form)
    if H is not None:
        Hx = np.asarray(H, np.float64)
    tb = tau(form, P['ldw'])
    if P['epi'] == 0:
        y = Hx.copy()
        b = np.zeros(P['N']) if 'bias' not in S else S['bias'].astype(np.float64)
        y += b
        e = e + tb * np.abs(b)
        if P['relu']:
            y = np.maximum(y, 0.0)
        r = S['res'].astype(np.float64) if 'res' in S else 0.0
        y = y + r
        return y, e + 2.0 ** -23 * (np.abs(y) + np.abs(r))
    if P['epi'] == 1:
        return _semch(P, S, Hx, e)
    return _global(P, S, Hx, e, tb)


def _semch(P, S, H, e):
    F, J, Cc, tpm = P['F'], P['J'], P['C'], P['tiles_per_mask']
    nm = nmasks(P)
    H, e = H.reshape(F, J, -1), e.reshape(F, J, -1)
    y = np.zeros((F, J, nm * Cc))
    bd = np.zeros_like(y)
    for m in range(nm):
        rp, col = P['nbr'][m]
        coef = S['coef'][m].astype(np.float64)
        sh = S['shift'][m * Cc:(m + 1) * Cc].astype(np.float64) if 'shift' in S else np.zeros(Cc)
        c = np.arange(Cc)
        self_col = (m * tpm + c // 64) * 128 + c % 64
        nbr_col = self_col + 64
        for i in range(J):
            acc = np.broadcast_to(sh, (F, Cc)).copy()
            err = np.zeros((F, Cc))
            mag = np.broadcast_to(np.abs(sh), (F, Cc)).copy()
            zs = range(rp[i], rp[i + 1])
            for z in zs:
                jj = col[z]
                hz, ez = (H[:, i, self_col], e[:, i, self_col]) if jj == i else (H[:, jj, nbr_col], e[:, jj, nbr_col])
                acc += coef[z] * hz
                err += np.abs(coef[z]) * ez
                mag += np.abs(coef[z]) * (np.abs(hz) + ez)
            if P['relu']:
                acc = np.maximum(acc, 0.0)
            y[:, i, m * Cc:(m + 1) * Cc] = acc
            bd[:, i, m * Cc:(m + 1) * Cc] = err + (len(zs) + 1) * U * mag
    return y.reshape(F * J, -1), bd.reshape(F * J, -1)


def attention(P, S):
    """(att64, eps): the attention rows (F, heads, J, J) in fp64 from the snapshot's ab and ck, and the relative
    bound of the device's fp32 softmax on each"""
    F, J, hd = P['F'], P['J'], P['heads']
    ab = S['ab'].astype(np.float64).reshape(F, J, 2 * hd)
    a, b = ab[:, :, 0::2], ab[:, :, 1::2]                      # (F, J, heads)
    s = a.transpose(0, 2, 1)[:, :, :, None] + b.transpose(0, 2, 1)[:, :, None, :]   # (F, heads, i, j)
    s = np.where(s >= 0, s, 0.2 * s)
    smax = np.abs(s).max(axis=3, keepdims=True)
    ex = np.exp(s - s.max(axis=3, keepdims=True))
    sm = ex / ex.sum(axis=3, keepdims=True)
    eps = 2 * (6 * smax * U + 2.0 ** -22) + (J + 2) * U
    att = sm + S['ck'].astype(np.float64)[None]
    return att, eps * sm + U * np.abs(att)


def _global(P, S, H, e, tb):
    F, J, N, Cg = P['F'], P['J'], P['N'], P['Cg']
    bg = S['bg'].astype(np.float64) if 'bg' in S else np.zeros(N)
    G = (H + bg).reshape(F, J, N)
    eG = (e + tb * np.abs(bg)).reshape(F, J, N)
    att, datt = attention(P, S)
    y = np.zeros((F, J, N))
    bd = np.zeros_like(y)
    for h in range(P['heads']):
        cs = slice(h * Cg, min((h + 1) * Cg, N))
        at, da = att[:, h], datt[:, h]
        y[:, :, cs] = np.einsum('fij,fjc->fic', at, G[:, :, cs])
        aa = np.abs(at)
        bd[:, :, cs] = (np.einsum('fij,fjc->fic', aa, eG[:, :, cs]) + np.einsum('fij,fjc->fic', da, np.abs(G[:, :, cs]))
                        + J * U * np.einsum('fij,fjc->fic', aa, np.abs(G[:, :, cs]) + eG[:, :, cs]))
    return y.reshape(F * J, N), bd.reshape(F * J, N)


def emulate(P, S, rows):
    """the tensor-core form's product on rows `rows` of the dense A (f16x3ref / tf32ref), float32"""
    A, W = S['A'][rows], S['W']
    if P['tc_form'] == 2:
        return F16.gemm(A, W)
    if P['tc_form'] == 0:
        return F16.gemm_3xtf32(A, W)
    return (TF.tf32(A).astype(np.float64) @ TF.tf32(W).astype(np.float64).T).astype(np.float32)


def _sub(P, S, rows):
    """(P, S) restricted to the frames of `rows` (for the emulation on a subset)"""
    fr = np.unique(rows // P['J'])
    r = (fr[:, None] * P['J'] + np.arange(P['J'])).ravel()
    P2 = dict(P, F=len(fr))
    S2 = dict(S, A=S['A'][r])
    for k in ('res', 'ab'):
        if k in S:
            S2[k] = S[k][r]
    return P2, S2, r


class AuditError(AssertionError):
    pass


def check(P, S, out1, form=None):
    """hold a launch's output (the window read after it ran) to the fp64 restatement; -> its record.  Raises
    AuditError naming the launch and the worst element when an element is past its bound, a column it does not own
    changed, or a tensor-core launch is off its form's emulation."""
    name = 'launch %d (%s, core %s, form %s, F %d J %d N %d K %d ld_out %d)' % (
        P['index'], EPI_NAMES[P['epi']], 'tc' if P['core'] == 0 else 'ffma', FORMS[P['tc_form']], P['F'], P['J'],
        P['N'], P['ldw'], P['ld_out'])
    w = width(P)
    y = out1[:, :w].astype(np.float64)
    y64, bd = restate(P, S, form)
    err = np.abs(y - y64)
    bad = ~np.isfinite(y)
    ratio = np.where(bd > 0, err / np.where(bd > 0, bd, 1.0), np.where(err > 0, np.inf, 0.0))
    ratio[bad] = np.inf
    worst = float(ratio.max()) if ratio.size else 0.0
    if worst > 1.0:
        r, c = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        raise AuditError('%s: element (%d, %d) = %r, fp64 %r, |err| %.3e > bound %.3e (%d elements past it)' % (
            name, r, c, float(y[r, c]), float(y64[r, c]), err[r, c], bd[r, c], int((ratio > 1).sum())))
    l2 = float(np.linalg.norm(y - y64) / max(np.linalg.norm(y64), 1e-300))
    # columns the launch does not own (all rows but the last, whose tail is past the window)
    tail0, tail1 = S['out0'][:-1, w:], out1[:-1, w:]
    if tail0.size and not np.array_equal(tail0.view(np.uint32), tail1.view(np.uint32)):
        r, c = np.argwhere(tail0.view(np.uint32) != tail1.view(np.uint32))[0]
        raise AuditError('%s: wrote column %d of row %d, past its %d columns (%r -> %r)' % (
            name, w + c, r, w, float(tail0[r, c]), float(tail1[r, c])))
    emu_l2 = None
    if P['core'] == 0:
        R = P['F'] * P['J']
        rows = np.arange(R) if R <= EMU_MAX_ROWS else np.unique(np.r_[np.linspace(0, R - 1, EMU_MAX_ROWS // 2).astype(
            np.int64), np.arange(R - EMU_MAX_ROWS // 2, R)])
        P2, S2, r = _sub(P, S, rows)
        ye, _ = restate(P2, S2, H=emulate(P2, S2, slice(None)))
        ye = ye.astype(np.float32).astype(np.float64)
        yr = y[r]
        emu_l2 = float(np.linalg.norm(yr - ye) / max(np.linalg.norm(ye), 1e-300))
        if emu_l2 > EMU_L2_BAR:
            raise AuditError('%s: relative L2 %.3e from the %s emulation (bar %.1e)' % (
                name, emu_l2, FORMS[P['tc_form']], EMU_L2_BAR))
    return dict(index=P['index'], epi=EPI_NAMES[P['epi']], core='tc' if P['core'] == 0 else 'ffma',
                form=FORMS[P['tc_form']], F=P['F'], J=P['J'], N=P['N'], K=P['ldw'], ld_out=P['ld_out'],
                tma_mask=P['tma_mask'], nseg=P['nseg'], worst=worst, l2=l2, emu_l2=emu_l2, shape=shape_tags(P))


def shape_tags(P):
    """the layout and epilogue features of a launch, for the coverage count"""
    t = set()
    R = P['F'] * P['J']
    t.add('nseg%d' % P['nseg'])
    if P['J'] == 1 and P['fpt'] == 128:
        t.add('flat')
    elif P['fpt'] * P['J'] < 128:
        t.add('frame_tiled')
    if R % (P['fpt'] * P['J']):
        t.add('partial_row_tile')
    if P['N'] % 128:
        t.add('partial_col_tile')
    if P['N'] < 32:
        t.add('N_lt_32')
    if R < 128:
        t.add('FJ_lt_128')
    if P['ld_out'] > width(P):
        t.add('ld_out_gt_N')
    if P['bias'] or (P['epi'] == 2 and P['bg']):
        t.add('bias')
    if P['relu']:
        t.add('relu')
    if P['epi'] == 0 and P['res']:
        t.add('res')
        if P['res_map'] != (1, 1, 1, 0) and P['res_map'][1:] != (P['res_map'][0], 1, 0):
            t.add('res_map')
    for s in P['segs']:
        if s['tap_stride'] and s['map'][2] > 1:
            t.add('tap_stride_t_mul')
        if s['tap_stride']:
            t.add('tap_stride')
        if s['map'][3]:
            t.add('t_off')
    if P['core'] == 0 and P['epi'] == 0:
        full = (1 << P['nseg']) - 1
        t.add('feed_tma' if P['tma_mask'] == full else 'feed_gather' if P['tma_mask'] == 0 else 'feed_mixed')
    return t


# ----------------------------------------------------------------------------------------------------------------
# the hook
# ----------------------------------------------------------------------------------------------------------------
class Auditor(object):
    """the callback of gast_debug_set_gemm_audit: snapshots each launch, checks it after it ran and keeps the records
    (self.records) and the first failure (self.failure, also returned to the library so that the call fails)"""

    def __init__(self, mem=None):
        from gast_b200 import _lib
        self.mem = mem or DeviceMemory()
        self.records = []
        self.failure = None
        self._pending = {}
        self.fn = _lib.GemmAuditFn(self._call)

    def _call(self, phase, d, user):
        try:
            P = params(d.contents)
            if phase == 0:
                self._pending[P['index']] = (P, snapshot(P, self.mem))
            else:
                P0, S = self._pending.pop(P['index'])
                self.records.append(check(P0, S, read_out(P0, self.mem)))
            return 0
        except Exception as ex:   # the library fails the call; the message is kept for the test
            if self.failure is None:
                import traceback
                self.failure = '%s: %s\n%s' % (type(ex).__name__, ex, traceback.format_exc(limit=-4))
            return 1

    def install(self, lib, h):
        rc = lib.gast_debug_set_gemm_audit(h, self.fn, None)
        assert rc == 0


def report_line(rec):
    return '%6d %-6s %-4s %-6s F %6d J %2d N %5d K %5d ld_out %5d tma %d worst %.3e l2 %.3e emu_l2 %s\n' % (
        rec['index'], rec['epi'], rec['core'], rec['form'], rec['F'], rec['J'], rec['N'], rec['K'], rec['ld_out'],
        rec['tma_mask'], rec['worst'], rec['l2'], '-' if rec['emu_l2'] is None else '%.3e' % rec['emu_l2'])


def write_report(lines, fname='gemm_audit.txt'):
    d = os.environ.get('GAST_TEST_REPORT_DIR')
    if d:
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, fname), 'a') as f:
            f.writelines(lines)

