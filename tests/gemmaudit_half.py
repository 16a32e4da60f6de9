"""Per-launch audit of the half form's GEMMs: each launch of a half forward (gast_set_activation_dtype(h, GAST_F16),
audit records with tc_form 3) held to fp64 of its own fp16 operands.

Test infrastructure, built on tests/gemmaudit.py (its record parsing, frame maps and the SemCH and global-attention
restatements).  What differs in half:
  * the A segments, the residual and the output window are fp16 in memory; W, bias, the SemCH coefficients and
    shift, the row dots, C_k and the `g` bias are fp32, as in every form;
  * the device multiplies by its fp16 weight copy fp16(W 2^s_W) 2^-s_W (s_W: max |W| 2^s_W in [2^14, 2^15),
    tc_wscale_kernel), so that copy is the W operand of the restatement;
  * K is chained in one fp32 accumulator: each k16 MMA truncates its 17 addends by less than one fp32 ulp of the
    largest, each at most the running sum of |a w|: |H^ - H| <= (K / 16) 17 2^-23 S, S = sum_k |a_k w_k| (the
    2^-s_W scale is exact);
  * the epilogue computes in fp32 (gemmaudit's bounds: the bias add u (S + |bias|), the residual add, the SemCH and
    attention chains), then rounds each stored value once to fp16: 2^-11 of its magnitude, or 2^-25 absolute among
    fp16's subnormals.
There is no separate emulation check: the bound above is already the fp32-accumulation bound of the fp16 products.
"""
import numpy as np

import gemmaudit as GA

U = GA.U
F16_HALF_ULP = 2.0 ** -11        # round to nearest fp16, relative
F16_SUB = 2.0 ** -25             # half the spacing of fp16's subnormals
FORM_HALF = 3


class DeviceMemory(GA.DeviceMemory):
    """fp32 spans (read) and fp16 spans widened to fp32 (read16) of device memory at raw addresses"""

    def read16(self, ptr, n):
        import torch

        class _Span(object):
            __cuda_array_interface__ = {'shape': (int(n),), 'typestr': '<f2', 'data': (int(ptr), False),
                                        'version': 2, 'strides': None}
        return torch.as_tensor(_Span(), device='cuda').cpu().numpy().astype(np.float32)


def _rows16(mem, base, offs, w):
    """rows of w halves at half offsets offs from base, from one span read -> offs.shape + (w,)"""
    offs = np.asarray(offs, np.int64)
    lo, hi = int(offs.min()), int(offs.max()) + w
    buf = mem.read16(base + 2 * lo, hi - lo)
    return buf[(offs - lo)[..., None] + np.arange(w)]


def gather_a(P, mem):
    """the dense fp16 A (F J, K) of the launch, segment by segment"""
    F, J = P['F'], P['J']
    f = np.repeat(np.arange(F), J)
    j = np.tile(np.arange(J), F)
    parts = []
    for s in P['segs']:
        taps = s['K'] // s['Kc']
        src = GA.map_frames(s['map'], f) * J + j
        offs = src[:, None] * s['ld'] + np.arange(taps)[None, :] * s['tap_stride']
        parts.append(_rows16(mem, s['base'], offs, s['Kc']).reshape(F * J, s['K']))
    return np.concatenate(parts, axis=1)


def weight_copy(W):
    """fp16(W 2^s_W) 2^-s_W in fp64: the weights the half form multiplies by"""
    W = np.asarray(W, np.float64)
    m = float(np.abs(W).max(initial=0.0))
    if m == 0.0 or not np.isfinite(m):
        return np.ldexp(W.astype(np.float16).astype(np.float64), 0)
    sw = 14 - (np.frexp(m)[1] - 1)
    return np.ldexp(np.ldexp(W, sw).astype(np.float16).astype(np.float64), -sw)


def read_out(P, mem):
    """the fp16 output window [0, F J) x [0, ld_out) up to the last element the launch writes, NaN-padded"""
    R, ld = P['F'] * P['J'], P['ld_out']
    n = (R - 1) * ld + GA.width(P)
    win = np.full(R * ld, np.nan, np.float32)
    win[:n] = mem.read16(P['out'], n)
    return win.reshape(R, ld)


def snapshot(P, mem):
    """the launch's operands and its output window, read before it runs"""
    F, J, N, K = P['F'], P['J'], P['N'], P['ldw']
    R = F * J
    S = {'A': gather_a(P, mem), 'W': mem.read(P['W'], N * K).reshape(N, K)}
    if P['bias']:
        S['bias'] = mem.read(P['bias'], N)
    if P['epi'] == 0 and P['res']:
        src = GA.map_frames(P['res_map'], np.repeat(np.arange(F), J)) * J + np.tile(np.arange(J), F)
        S['res'] = _rows16(mem, P['res'], src * P['res_ld'], N)
    if P['epi'] == 1:
        nm = GA.nmasks(P)
        S['coef'] = [mem.read(P['coef'][m], GA.nnz(P, m) * P['C']).reshape(-1, P['C']) for m in range(nm)]
        if P['shift']:
            S['shift'] = mem.read(P['shift'], nm * P['C'])
    if P['epi'] == 2:
        S['ab'] = mem.read(P['ab'], R * 2 * P['heads']).reshape(R, 2 * P['heads'])
        S['ck'] = mem.read(P['ck'], P['heads'] * J * J).reshape(P['heads'], J, J)
        if P['bg']:
            S['bg'] = mem.read(P['bg'], N)
    S['out0'] = read_out(P, mem)
    return S


def restate(P, S):
    """(y64, bound): the launch's output columns [0, width) in fp64 from its fp16 operands and the elementwise bound
    of the half form (module docstring)"""
    A = S['A'].astype(np.float64)
    W = weight_copy(S['W'])
    H = A @ W.T
    K = A.shape[1]
    mag = np.abs(A) @ np.abs(W).T
    e = ((K / 16.0) * 17 * 2.0 ** -23 + U) * mag          # accumulation, and the bias add's rounding on S
    if P['epi'] == 0:
        b = np.zeros(P['N']) if 'bias' not in S else S['bias'].astype(np.float64)
        y = H + b
        e = e + U * np.abs(b)
        if P['relu']:
            y = np.maximum(y, 0.0)
        r = S['res'].astype(np.float64) if 'res' in S else 0.0
        y = y + r
        e = e + 2.0 ** -23 * (np.abs(y) + np.abs(r))
    elif P['epi'] == 1:
        y, e = GA._semch(P, S, H, e)
    else:
        y, e = GA._global(P, S, H, e, U)
    return y, e + F16_HALF_ULP * (np.abs(y) + e) + F16_SUB


def check(P, S, out1):
    """hold a half launch's fp16 output to its fp64 restatement; -> its record.  Raises gemmaudit.AuditError naming
    the launch and the worst element, or a column past the launch's width that changed."""
    assert P['tc_form'] == FORM_HALF and P['core'] == 0, (P['tc_form'], P['core'])
    name = 'launch %d (%s, half, F %d J %d N %d K %d ld_out %d)' % (
        P['index'], GA.EPI_NAMES[P['epi']], P['F'], P['J'], P['N'], P['ldw'], P['ld_out'])
    w = GA.width(P)
    y = out1[:, :w].astype(np.float64)
    y64, bd = restate(P, S)
    err = np.abs(y - y64)
    ratio = err / bd
    ratio[~np.isfinite(y)] = np.inf
    worst = float(ratio.max()) if ratio.size else 0.0
    if worst > 1.0:
        r, c = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
        raise GA.AuditError('%s: element (%d, %d) = %r, fp64 %r, |err| %.3e > bound %.3e (%d elements past it)' % (
            name, r, c, float(y[r, c]), float(y64[r, c]), err[r, c], bd[r, c], int((ratio > 1).sum())))
    tail0, tail1 = S['out0'][:-1, w:], out1[:-1, w:]
    if tail0.size and not np.array_equal(tail0.view(np.uint32), tail1.view(np.uint32)):
        r, c = np.argwhere(tail0.view(np.uint32) != tail1.view(np.uint32))[0]
        raise GA.AuditError('%s: wrote column %d of row %d, past its %d columns' % (name, w + c, r, w))
    rel = float(np.abs(y - y64).max() / max(np.abs(y64).max(), 1e-300))
    return dict(index=P['index'], epi=GA.EPI_NAMES[P['epi']], F=P['F'], J=P['J'], N=P['N'], K=P['ldw'],
                tma_mask=P['tma_mask'], nseg=P['nseg'], worst=worst, max_rel=rel, shape=GA.shape_tags(P))


class Auditor(GA.Auditor):
    """gemmaudit.Auditor for the launches of a half forward"""

    def __init__(self):
        super(Auditor, self).__init__(DeviceMemory())

    def _call(self, phase, d, user):
        try:
            P = GA.params(d.contents)
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
