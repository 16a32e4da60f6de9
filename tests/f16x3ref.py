"""numpy emulation of the tensor-core core's fp32-grade inference form (F16X3, csrc/gemm_tc.cuh) and, for comparison,
of the 3xTF32 form training runs.

Test infrastructure, CPU only.  F16X3 scales W by 2^s_W (one exponent per matrix, max |W| 2^s_W in [2^14, 2^15)) and
each A row by 2^s_r per 32-K stage (the same rule on the row's 32 values), splits both into fp16 hi / lo and sums
A_lo.B_hi + A_hi.B_lo + A_hi.B_hi per 16-K partial; the partial is added into the fp32 tile sum times
2^-(s_r + s_W).  The splits and scales here are the device's bit for bit; the products of a partial are summed in fp64
(the tensor core sums them in fp32 with truncation), so a GEMM through `gemm` is an emulation, not a bitwise copy.
"""
import numpy as np

from tf32ref import tf32

KS, KP = 32, 16          # K per ring stage (one row scale each), K per partial sum
F16_MAX = 65504.0


def w_scale(W):
    """s_W: max |W| 2^s_W in [2^14, 2^15); 0 for an all-zero or non-finite W (tc_wscale_kernel)"""
    m = np.float32(np.fmax.reduce(np.abs(np.asarray(W, np.float32)).ravel(), initial=np.float32(0)))
    if m == 0 or not np.isfinite(m):
        return 0
    return 14 - (int(np.frexp(m)[1]) - 1)


def scale_bounds(sw):
    """s_r's range, so that 2^s_r and 2^-(s_r + s_W) are both normal fp32 (tc_scale_bounds)"""
    return max(-126, -127 - sw), min(127, 126 - sw)


def row_scales(A, sw):
    """s_r of every row and 32-K stage of A (M, K) -> (M, K / 32) int: from the biased exponent of the row's max |a|
    (NaN ignored, as fmaxf does), 0 for a zero or infinite max, clamped (tc_row_exp)"""
    A = np.asarray(A, np.float32)
    M, K = A.shape
    m = np.fmax.reduce(np.abs(A).reshape(M, K // KS, KS), axis=2, initial=np.float32(0)).astype(np.float32)
    eb = (m.view(np.uint32) >> np.uint32(23)).astype(np.int64)
    s = np.where((m == 0) | (eb == 255), 0, 141 - eb)
    lo, hi = scale_bounds(sw)
    return np.clip(s, lo, hi)


def pow2(e):
    """2^e as float32, e an int array in [-126, 127]"""
    return np.ldexp(np.float32(1), np.asarray(e)).astype(np.float32)


def split16(x):
    """fp32 x -> (fp16(x), fp16(x - fp16(x))), round to nearest even (cvt.rn.f16x2.f32)"""
    x = np.asarray(x, np.float32)
    with np.errstate(over='ignore', invalid='ignore'):
        h = x.astype(np.float16)
        lo = (x - h.astype(np.float32)).astype(np.float16)
    return h, lo


def split_w(W):
    """(hi, lo, s_W) of a weight matrix, as tc_split16_kernel stores them"""
    W = np.asarray(W, np.float32)
    sw = w_scale(W)
    h, lo = split16(np.ldexp(W, sw).astype(np.float32))
    return h, lo, sw


def split_a(A, sw):
    """(hi, lo, s) of A's rows: hi, lo (M, K) fp16 of A 2^s_r stage by stage, s (M, K / 32) the s_r"""
    A = np.asarray(A, np.float32)
    s = row_scales(A, sw)
    scaled = (A * np.repeat(pow2(s), KS, axis=1)).astype(np.float32)   # exact but where it lands subnormal
    h, lo = split16(scaled)
    return h, lo, s


def _accumulate(parts, scales):
    """fp32 tile sum of per-partial fp64 products: acc = fp32(acc + fp32(part) * scale)"""
    acc = None
    for part, u in zip(parts, scales):
        p = part.astype(np.float32).astype(np.float64) * u
        acc = p.astype(np.float32) if acc is None else (acc.astype(np.float64) + p).astype(np.float32)
    return acc


def gemm(A, W):
    """A (M, K) . W (N, K)^T in the F16X3 form -> (M, N) float32"""
    A, W = np.asarray(A, np.float32), np.asarray(W, np.float32)
    wh, wl, sw = split_w(W)
    ah, al, s = split_a(A, sw)
    f = lambda x: x.astype(np.float64)   # noqa: E731
    parts, scales = [], []
    with np.errstate(invalid='ignore', over='ignore'):
        for k in range(0, A.shape[1], KP):
            sl = slice(k, k + KP)
            parts.append(f(al[:, sl]) @ f(wh[:, sl]).T + f(ah[:, sl]) @ f(wl[:, sl]).T + f(ah[:, sl]) @ f(wh[:, sl]).T)
            scales.append(f(pow2(-(s[:, k // KS] + sw)))[:, None])
        return _accumulate(parts, scales)


def gemm_3xtf32(A, W):
    """A (M, K) . W (N, K)^T in the 3xTF32 form, with the same partials and accumulation -> (M, N) float32"""
    A, W = np.asarray(A, np.float32), np.asarray(W, np.float32)
    ah, wh = tf32(A), tf32(W)
    al, wl = tf32(A - ah), tf32(W - wh)
    f = lambda x: x.astype(np.float64)   # noqa: E731
    parts = []
    for k in range(0, A.shape[1], KP):
        sl = slice(k, k + KP)
        parts.append(f(al[:, sl]) @ f(wh[:, sl]).T + f(ah[:, sl]) @ f(wl[:, sl]).T + f(ah[:, sl]) @ f(wh[:, sl]).T)
    return _accumulate(parts, [1.0] * len(parts))
