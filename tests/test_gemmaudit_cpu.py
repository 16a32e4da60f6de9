"""CPU checks of the per-launch GEMM audit (tests/gemmaudit.py) without a GPU.

Launches are laid out in a host address space (HostMemory) whose reads fail outside a buffer, so the snapshot is also
held to reading only inside the allocations a launch touches.
  * The vectorised fp64 restatement against a per-element loop over the same definitions, on random launches with 1 to
    3 segments, temporal taps, strided and offset frame maps, a residual map, ld_out > N, partial row and column tiles,
    and SemCH and global-attention tiles at J = 15 and 19.
  * Launches built from the torch port's layers against float64 torch (the stage convolution of
    oracle/gast_torch_ref.py forward with dilation or stride and its residual slice, the 1x1 layer, the block
    concatenation).
  * Teeth: the checker fails a snapshot changed on the host only -- one element of a partial column tile's tail column
    off by 16 ulp, one frame-tile row replaced by the next frame's, one value written into column N of an ld_out > N
    window, a 1xTF32 result held to the fp32-grade bound -- and passes each unchanged one.
"""
import math

import numpy as np
import pytest
import torch

import gemmaudit as G
import f16x3ref as F16
import tf32ref as TF


class HostMemory(object):
    """numpy buffers at fake, 256-byte-aligned addresses with gaps between them; a read must stay in one buffer"""

    def __init__(self):
        self.bufs = []
        self.next = 1 << 20

    def add(self, a):
        a = np.ascontiguousarray(a, np.float32).ravel()
        base = self.next
        self.bufs.append((base, a))
        self.next += ((a.size * 4 + 255) // 256 + 4) * 256
        return base

    def _find(self, ptr):
        for base, a in self.bufs:
            if base <= ptr < base + 4 * a.size:
                return base, a
        raise AssertionError('read at 0x%x is in no allocation' % ptr)

    def read(self, ptr, n):
        base, a = self._find(ptr)
        off = (ptr - base) // 4
        assert (ptr - base) % 4 == 0 and off + n <= a.size, 'read of %d floats at 0x%x runs past its allocation' % (
            n, ptr)
        return a[off:off + n].copy()

    def at(self, ptr):
        return float(self.read(ptr, 1)[0])


IDENT = (1, 1, 1, 0)


def base_params(F, J, fpt, N, K, ld_out, epi=0, form=-1):
    return dict(index=0, epi=epi, core=1 if form < 0 else 0, tc_form=form, tma_mask=0, nseg=0, ldw=K, N=N, F=F, J=J,
                fpt=fpt, ld_out=ld_out, relu=0, res_ld=0, C=0, tiles_per_mask=0, heads=0, Cg=0, segs=[], W=0, out=0,
                bias=0, res=0, shift=0, ab=0, ck=0, bg=0, coef=[0, 0], res_map=IDENT, nbr=[([0] * 36, [0] * 164)] * 2)


def add_seg(P, mem, rs, Kc, taps, T_in, T_out, t_mul, t_off, dil, J, extra_cols=0):
    """a segment over a fresh source of B clips of T_in frames; taps dil frames apart"""
    B = P['F'] // T_out
    ld = Kc + extra_cols
    src = rs.standard_normal((B * T_in * J, ld)).astype(np.float32)
    P['segs'].append(dict(base=mem.add(src), ld=ld, K=taps * Kc, Kc=Kc, tap_stride=dil * J * ld,
                          map=(T_out, T_in, t_mul, t_off)))
    P['nseg'] += 1
    return src


def nbr_table(J, rs, self_loops=True):
    """a random row-major neighbour table (every row non-empty)"""
    rp, col = [0] * 36, [0] * 164
    z = 0
    for i in range(J):
        rp[i] = z
        cols = sorted(set(rs.choice(J, 3, replace=False).tolist()) | ({i} if self_loops else set()))
        for c in cols:
            col[z] = c
            z += 1
    rp[J] = z
    return rp, col


def plain_launch(rs, nseg=2, J=17, fpt=7, T_out=5, B=3, N=132, relu=1, res=True, ld_extra=8, taps=(3, 1, 2),
                 form=-1):
    mem = HostMemory()
    F = B * T_out
    P = base_params(F, J, fpt, N, 0, N + ld_extra, form=form)
    # segment s: (T_in, t_mul, t_off, dilation): a strided tap conv, an identity map, an offset dilated tap conv
    for s in range(nseg):
        T_in, t_mul, t_off, dil = [(T_out * 3 + 2, 3, 0, 1), (T_out, 1, 0, 1), (T_out + 6, 1, 2, 3)][s]
        add_seg(P, mem, rs, 8 * (s + 1), taps[s], T_in, T_out, t_mul, t_off, dil, J, extra_cols=4 * s)
    K = sum(s['K'] for s in P['segs'])
    P['ldw'] = K
    P['W'] = mem.add((rs.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32))
    P['bias'] = mem.add(rs.standard_normal(N).astype(np.float32))
    P['relu'] = relu
    if res:
        T_rin = T_out * 2 + 3
        P['res'] = mem.add(rs.standard_normal((B * T_rin * J, N + 4)).astype(np.float32))
        P['res_ld'] = N + 4
        P['res_map'] = (T_out, T_rin, 2, 1)
    P['out'] = mem.add(np.full((F * J, P['ld_out']), 7.0, np.float32))
    return P, mem


def semch_launch(rs, J, Cc=36, Cin=32, F=9, fpt=None, nmask=2, relu=1):
    mem = HostMemory()
    tpm = (Cc + 63) // 64
    N = nmask * tpm * 128
    P = base_params(F, J, fpt or 128 // J, N, Cin, nmask * Cc, epi=1)
    add_seg(P, mem, rs, Cin, 1, 1, 1, 1, 0, 0, J)
    P['W'] = mem.add((rs.standard_normal((N, Cin)) / np.sqrt(Cin)).astype(np.float32))
    P['C'], P['tiles_per_mask'], P['relu'] = Cc, tpm, relu
    nbr = [nbr_table(J, rs, self_loops=(m == 0)) for m in range(nmask)] + [([0] * 36, [0] * 164)] * (2 - nmask)
    P['nbr'] = nbr
    P['coef'] = [mem.add(rs.standard_normal((nbr[m][0][J], Cc)).astype(np.float32)) if m < nmask else 0
                 for m in range(2)]
    P['shift'] = mem.add(rs.standard_normal(nmask * Cc).astype(np.float32))
    P['out'] = mem.add(np.zeros((F * J, nmask * Cc), np.float32))
    return P, mem


def global_launch(rs, J, heads=3, Cg=12, Cin=32, F=8):
    mem = HostMemory()
    N = heads * Cg
    P = base_params(F, J, 128 // J, N, Cin, N, epi=2)
    P['segs'].append(dict(base=mem.add(rs.standard_normal((F * J, Cin)).astype(np.float32)), ld=Cin, K=Cin, Kc=Cin,
                          tap_stride=0, map=IDENT))
    P['nseg'] = 1
    P['W'] = mem.add((rs.standard_normal((N, Cin)) / np.sqrt(Cin)).astype(np.float32))
    P['heads'], P['Cg'] = heads, Cg
    P['ab'] = mem.add(rs.standard_normal((F * J, 2 * heads)).astype(np.float32))
    P['ck'] = mem.add((0.1 * rs.standard_normal((heads, J, J))).astype(np.float32))
    P['bg'] = mem.add(rs.standard_normal(N).astype(np.float32))
    P['out'] = mem.add(np.zeros((F * J, N), np.float32))
    return P, mem


# ----------------------------------------------------------------------------------------------------------------
# the brute-force restatement: one element at a time, straight from the definitions
# ----------------------------------------------------------------------------------------------------------------
def _map(m, f):
    T_out, T_in, t_mul, t_off = m
    return (f // T_out) * T_in + (f % T_out) * t_mul + t_off


def brute_h(P, mem, r, n):
    f, j = divmod(r, P['J'])
    terms, kcol = [], 0
    for s in P['segs']:
        src = _map(s['map'], f) * P['J'] + j
        for k in range(s['K']):
            tap, c = divmod(k, s['Kc'])
            a = mem.at(s['base'] + 4 * (src * s['ld'] + tap * s['tap_stride'] + c))
            w = mem.at(P['W'] + 4 * (n * P['ldw'] + kcol + k))
            terms.append(a * w)
        kcol += s['K']
    return math.fsum(terms)


def brute(P, mem):
    F, J, N = P['F'], P['J'], P['N']
    R = F * J
    if P['epi'] == 0:
        y = np.zeros((R, N))
        for r in range(R):
            f, j = divmod(r, J)
            for n in range(N):
                v = brute_h(P, mem, r, n) + (mem.at(P['bias'] + 4 * n) if P['bias'] else 0.0)
                if P['relu']:
                    v = max(v, 0.0)
                if P['res']:
                    v += mem.at(P['res'] + 4 * ((_map(P['res_map'], f) * J + j) * P['res_ld'] + n))
                y[r, n] = v
        return y
    if P['epi'] == 1:
        Cc, tpm = P['C'], P['tiles_per_mask']
        nm = N // (128 * tpm)
        y = np.zeros((R, nm * Cc))
        for r in range(R):
            f, i = divmod(r, J)
            for m in range(nm):
                rp, col = P['nbr'][m]
                for c in range(Cc):
                    t, cl = divmod(c, 64)
                    tile = m * tpm + t
                    v = [mem.at(P['shift'] + 4 * (m * Cc + c))] if P['shift'] else []
                    for z in range(rp[i], rp[i + 1]):
                        jj = col[z]
                        h = brute_h(P, mem, r, tile * 128 + cl) if jj == i else brute_h(P, mem, f * J + jj,
                                                                                       tile * 128 + 64 + cl)
                        v.append(mem.at(P['coef'][m] + 4 * (z * Cc + c)) * h)
                    s = math.fsum(v)
                    y[r, m * Cc + c] = max(s, 0.0) if P['relu'] else s
        return y
    hd = 2 * P['heads']
    y = np.zeros((R, N))
    for f in range(F):
        G = np.array([[brute_h(P, mem, f * J + j, n) + mem.at(P['bg'] + 4 * n) for n in range(N)] for j in range(J)])
        for h in range(P['heads']):
            for i in range(J):
                a = mem.at(P['ab'] + 4 * ((f * J + i) * hd + 2 * h))
                s = [a + mem.at(P['ab'] + 4 * ((f * J + j) * hd + 2 * h + 1)) for j in range(J)]
                s = [v if v >= 0 else 0.2 * v for v in s]
                mx = max(s)
                e = [math.exp(v - mx) for v in s]
                tot = math.fsum(e)
                att = [e[j] / tot + mem.at(P['ck'] + 4 * ((h * J + i) * J + j)) for j in range(J)]
                for n in range(h * P['Cg'], min((h + 1) * P['Cg'], N)):
                    y[f * J + i, n] = math.fsum(att[j] * G[j, n] for j in range(J))
    return y


CASES = {
    'plain_1seg_taps_strided': lambda rs: plain_launch(rs, nseg=1, N=36),
    'plain_2seg_offset_res': lambda rs: plain_launch(rs, nseg=2, N=132),
    'plain_3seg_flat_partial': lambda rs: plain_launch(rs, nseg=3, J=1, fpt=128, T_out=40, B=4, N=20, relu=0),
    'plain_3seg_j19_no_res': lambda rs: plain_launch(rs, nseg=3, J=19, fpt=6, N=136, res=False),
    'semch_j15': lambda rs: semch_launch(rs, 15, Cc=36),
    'semch_j19_wide': lambda rs: semch_launch(rs, 19, Cc=68, F=4, relu=0),
    'semch_j19_one_mask': lambda rs: semch_launch(rs, 19, Cc=20, F=5, nmask=1),
    'global_j15': lambda rs: global_launch(rs, 15),
    'global_j19': lambda rs: global_launch(rs, 19, heads=4, Cg=8, F=6),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_restatement_matches_brute_force(name):
    rs = np.random.RandomState(sorted(CASES).index(name) + 1)
    P, mem = CASES[name](rs)
    S = G.snapshot(P, mem)
    y, bd = G.restate(P, S)
    yb = brute(P, mem)
    assert y.shape == yb.shape == (P['F'] * P['J'], G.width(P))
    np.testing.assert_allclose(y, yb, rtol=1e-12, atol=1e-12 * np.abs(yb).max())
    assert np.all(bd > 0)
    # the correctly rounded fp32 result is an FFMA launch's best case: it passes, and so do its untouched columns
    out1 = S['out0'].copy()
    out1[:, :G.width(P)] = y.astype(np.float32)
    rec = G.check(P, S, out1)
    assert rec['worst'] < 0.6, rec


def test_snapshot_stays_inside_allocations():
    """an output that is the right half of a buffer twice its width (ld_out = 2 N): the last row's window ends at the
    buffer's end, and the snapshot reads no further"""
    rs = np.random.RandomState(3)
    P, mem = plain_launch(rs, nseg=1, N=36, ld_extra=0, res=False)
    R, N = P['F'] * P['J'], P['N']
    buf = np.zeros((R, 2 * N), np.float32)
    P['out'] = mem.add(buf) + 4 * N
    P['ld_out'] = 2 * N
    S = G.snapshot(P, mem)
    assert S['out0'].shape == (R, 2 * N) and np.isnan(S['out0'][-1, N:]).all()
    P['out'] += 4
    with pytest.raises(AssertionError, match='past its allocation'):
        G.snapshot(P, mem)


# ----------------------------------------------------------------------------------------------------------------
# against float64 torch on the port's layers
# ----------------------------------------------------------------------------------------------------------------
def _cl(x):
    """(B, C, T, J) -> channels-last rows (B T J, C)"""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1]).contiguous().numpy()


@pytest.mark.parametrize('strided,causal', [(False, False), (True, False), (False, True), (True, True)])
def test_stage_against_torch(strided, causal):
    """one temporal stage of gast_torch_ref.forward (conv over fw taps, dilated by nd or strided by fw, then the 1x1
    layer and the residual slice), as the two launches run_stage makes, against float64 torch"""
    rs = np.random.RandomState(11 + 2 * strided + causal)
    B, Cw, J, fw, nd, T = 2, 32, 15, 3, 3, 31
    x = torch.from_numpy(rs.standard_normal((B, Cw, T, J)).astype(np.float32))
    w0 = torch.from_numpy((rs.standard_normal((Cw, Cw, fw, 1)) / 10).astype(np.float32))
    w1 = torch.from_numpy((rs.standard_normal((Cw, Cw, 1, 1)) / 6).astype(np.float32))
    b0 = torch.from_numpy(rs.standard_normal(Cw).astype(np.float32))
    b1 = torch.from_numpy(rs.standard_normal(Cw).astype(np.float32))
    pad = (fw - 1) * nd // 2
    if strided:
        shift = fw // 2 if causal else 0
        g = dict(stride=(fw, 1))
        res = x[:, :, shift + fw // 2::fw]
        dil, t_mul, res_mul, res_off = 1, fw, fw, shift + fw // 2
    else:
        shift = fw // 2 * nd if causal else 0
        g = dict(dilation=(nd, 1))
        res = x[:, :, pad + shift:T - pad + shift]
        dil, t_mul, res_mul, res_off = nd, 1, 1, pad + shift
    x64 = x.double()
    tmp64 = torch.relu(torch.nn.functional.conv2d(x64, w0.double(), b0.double(), **g))
    T_out = tmp64.shape[2]
    out64 = res.double()[:, :, :T_out] + torch.relu(torch.nn.functional.conv2d(tmp64, w1.double(), b1.double()))
    assert res.shape[2] == T_out
    mem = HostMemory()
    F = B * T_out
    P = base_params(F, J, 128 // J, Cw, fw * Cw, Cw)
    P['segs'] = [dict(base=mem.add(_cl(x)), ld=Cw, K=fw * Cw, Kc=Cw, tap_stride=dil * J * Cw, map=(T_out, T, t_mul, 0))]
    P['nseg'] = 1
    P['W'] = mem.add(w0[:, :, :, 0].permute(0, 2, 1).reshape(Cw, fw * Cw).numpy())   # tap-major K
    P['bias'], P['relu'], P['out'] = mem.add(b0.numpy()), 1, mem.add(np.zeros((F * J, Cw)))
    y0, _ = G.restate(P, G.snapshot(P, mem))
    np.testing.assert_allclose(y0, _cl(tmp64), rtol=1e-12, atol=1e-12)
    tmp = torch.from_numpy(y0.astype(np.float32))
    mem2 = HostMemory()
    P1 = base_params(F, J, 128 // J, Cw, Cw, Cw)
    P1['segs'] = [dict(base=mem2.add(tmp.numpy()), ld=Cw, K=Cw, Kc=Cw, tap_stride=0, map=IDENT)]
    P1['nseg'] = 1
    P1['W'] = mem2.add(w1[:, :, 0, 0].numpy())
    P1['bias'], P1['relu'], P1['out'] = mem2.add(b1.numpy()), 1, mem2.add(np.zeros((F * J, Cw)))
    P1['res'], P1['res_ld'], P1['res_map'] = mem2.add(_cl(x)), Cw, (T_out, T, res_mul, res_off)
    y1, _ = G.restate(P1, G.snapshot(P1, mem2))
    tmp_f = tmp.double().reshape(B, T_out, J, Cw).permute(0, 3, 1, 2)
    ref1 = res.double() + torch.relu(torch.nn.functional.conv2d(tmp_f, w1.double(), b1.double()))
    np.testing.assert_allclose(y1, _cl(ref1), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(y1, _cl(out64), rtol=1e-5, atol=1e-5)   # through the fp32 intermediate


def test_block_concatenation_against_torch():
    """the block's cat conv (gast_torch_ref.graph_attention_block): three segments from three buffers, run flat"""
    rs = np.random.RandomState(5)
    B, Cc, T, J = 2, 32, 4, 17
    parts = [torch.from_numpy(rs.standard_normal((B, Cc, T, J)).astype(np.float32)) for _ in range(3)]
    w = torch.from_numpy((rs.standard_normal((2 * Cc, 3 * Cc, 1, 1)) / 10).astype(np.float32))
    b = torch.from_numpy(rs.standard_normal(2 * Cc).astype(np.float32))
    ref = torch.relu(torch.nn.functional.conv2d(torch.cat([p.double() for p in parts], 1), w.double(), b.double()))
    mem = HostMemory()
    R = B * T * J
    P = base_params(R, 1, 128, 2 * Cc, 3 * Cc, 2 * Cc)
    P['segs'] = [dict(base=mem.add(_cl(p)), ld=Cc, K=Cc, Kc=Cc, tap_stride=0, map=IDENT) for p in parts]
    P['nseg'] = 3
    P['W'], P['bias'], P['relu'] = mem.add(w[:, :, 0, 0].numpy()), mem.add(b.numpy()), 1
    P['out'] = mem.add(np.zeros((R, 2 * Cc)))
    y, _ = G.restate(P, G.snapshot(P, mem))
    np.testing.assert_allclose(y, _cl(ref), rtol=1e-12, atol=1e-12)


# ----------------------------------------------------------------------------------------------------------------
# teeth
# ----------------------------------------------------------------------------------------------------------------
def _ffma_out(P, S):
    out1 = S['out0'].copy()
    y, _ = G.restate(P, S)
    out1[:, :G.width(P)] = y.astype(np.float32)
    return out1


def test_tail_column_16_ulp_fails():
    """an FFMA launch over K = 8 with non-negative operands (sum |a w| = |y|, so its bound is a few ulp): one element
    of column 130, in the 4-column tail of the second column tile, 16 ulp off"""
    rs = np.random.RandomState(21)
    mem = HostMemory()
    J, F, N, K = 17, 14, 132, 8
    P = base_params(F, J, 7, N, K, N)
    P['segs'] = [dict(base=mem.add(rs.uniform(0.5, 2, (F * J, K))), ld=K, K=K, Kc=K, tap_stride=0, map=IDENT)]
    P['nseg'] = 1
    P['W'] = mem.add(rs.uniform(0.5, 2, (N, K)))
    P['out'] = mem.add(np.zeros((F * J, N), np.float32))
    S = G.snapshot(P, mem)
    out1 = _ffma_out(P, S)
    G.check(P, S, out1)
    out1.view(np.uint32)[100, 130] += 16
    with pytest.raises(G.AuditError, match=r'element \(100, 130\)'):
        G.check(P, S, out1)


def test_row_from_next_frame_fails():
    rs = np.random.RandomState(22)
    P, mem = plain_launch(rs, nseg=2, N=36)
    S = G.snapshot(P, mem)
    out1 = _ffma_out(P, S)
    G.check(P, S, out1)
    J = P['J']
    f = 6                                      # the last frame of the first 7-frame tile
    out1[f * J + 3] = out1[(f + 1) * J + 3]
    with pytest.raises(G.AuditError, match=r'element \(%d, ' % (f * J + 3)):
        G.check(P, S, out1)


def test_write_into_column_n_fails():
    rs = np.random.RandomState(23)
    P, mem = plain_launch(rs, nseg=1, N=36, ld_extra=8)
    S = G.snapshot(P, mem)
    out1 = _ffma_out(P, S)
    G.check(P, S, out1)
    out1[40, P['N']] = 0.0
    with pytest.raises(G.AuditError, match='wrote column 36 of row 40'):
        G.check(P, S, out1)


def test_tf32_held_to_fp32_grade_bound_fails():
    """a 1xTF32 tensor-core launch's result (its emulation) passes its own bound and fails the 3xTF32 one"""
    rs = np.random.RandomState(24)
    mem = HostMemory()
    R, N, K = 256, 64, 128
    P = base_params(R, 1, 128, N, K, N, form=1)
    A = rs.standard_normal((R, K)).astype(np.float32)
    W = (rs.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    P['segs'] = [dict(base=mem.add(A), ld=K, K=K, Kc=K, tap_stride=0, map=IDENT)]
    P['nseg'], P['tma_mask'] = 1, 1
    P['W'] = mem.add(W)
    P['out'] = mem.add(np.zeros((R, N), np.float32))
    S = G.snapshot(P, mem)
    out1 = (TF.tf32(A).astype(np.float64) @ TF.tf32(W).astype(np.float64).T).astype(np.float32)
    rec = G.check(P, S, out1)
    assert rec['worst'] < 0.5 and rec['emu_l2'] < 1e-7, rec
    with pytest.raises(G.AuditError, match='past it'):
        G.check(P, S, out1, form=0)
    # and the fp32-grade forms' own emulations pass their bound
    for form, emu in ((0, F16.gemm_3xtf32), (2, F16.gemm)):
        P2 = dict(P, tc_form=form)
        rec = G.check(P2, S, emu(A, W))
        assert rec['worst'] < 0.5 and rec['emu_l2'] < 1e-9, rec


def test_tau_orders():
    """the forms' bounds in the order of their arithmetic"""
    K = 1536
    assert G.tau(1, K) > 50 * G.tau(0, K)
    assert G.tau(-1, K) > G.tau(0, K) > G.tau(2, K) > 2.0 ** -20
