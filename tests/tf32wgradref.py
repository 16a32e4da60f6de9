"""numpy emulation of the TF32 weight-gradient kernel (csrc/wgrad_tc.cuh) and of the kernel choice of dense_tn
(csrc/train.cuh) in the TF32 training precision.

Test infrastructure, CPU only.  dW[N][K] = sum over the rows m of dZ[m][N] . A[m][K]:
  - both operands rounded to tf32 (cvt.rna.tf32.f32: nearest, ties away from zero, 10 mantissa bits), restated here
    in floating-point arithmetic so that tests/test_tf32_wgrad_cpu.py can hold it against tests/tf32ref.py's bit trick;
  - the rows split into dense_tn's row ranges, each range's products summed exactly (fp64) and rounded to fp32 once:
    the kernel's fp32 accumulation of tf32 products differs from that by accumulation rounding only;
  - the fp32 partials summed in split order, as wgrad_reduce_kernel sums them.
"""
import numpy as np

WG_T, WG_M = 128, 16      # tile edge and row step of dense_tn's split (train_kernels.cuh)


def tf32(x):
    """round fp32(x) to nearest tf32, ties away from zero (fp32 subnormals at their fixed quantum 2^-136).  Inf and NaN
    pass through; values that round past the largest finite fp32 become inf, as in the hardware."""
    f = np.asarray(x, dtype=np.float32).astype(np.float64)
    out = f.copy()
    fin = np.isfinite(f) & (f != 0)
    m, e = np.frexp(f[fin])                              # |f| = m 2^e, m in [0.5, 1)
    q = np.ldexp(1.0, np.maximum(e, -125) - 11)          # quantum: 11 significant bits, fixed below 2^-126
    a = np.abs(f[fin])
    out[fin] = np.sign(f[fin]) * np.floor(a / q + 0.5) * q
    with np.errstate(over='ignore'):
        return out.astype(np.float32)


def split(M, N, K, sms):
    """(row splits, rows per split) of dense_tn for M rows on a device with `sms` multiprocessors"""
    tiles = -(-N // WG_T) * -(-K // WG_T)
    S = max(1, min(-(-M // 256), -(-2 * sms // tiles)))
    rps = -(-(-(-M // S)) // WG_M) * WG_M
    return max(1, -(-M // rps)), rps


def takes(N, K):
    """whether wgrad_tc_kernel takes a contraction with N dW rows and K dW columns (dense, aligned operands)"""
    return N % 32 == 0 and K % 32 == 0


def wgrad(dZ, A, sms):
    """the emulated TF32 weight gradient dZ^T . A (float32 [N][K])"""
    M, N = dZ.shape
    K = A.shape[1]
    S, rps = split(M, N, K, sms)
    z = tf32(dZ).astype(np.float64)
    a = tf32(A).astype(np.float64)
    out = np.zeros((N, K), np.float32)
    for s in range(S):
        part = (z[s * rps:(s + 1) * rps].T @ a[s * rps:(s + 1) * rps]).astype(np.float32)
        out = out + part                                 # fp32 adds, in split order
    return out


def bound(dZ, A, sms):
    """elementwise bound on |wgrad - exact dZ^T . A|: operand rounding (2^-11 relative each, both operands) plus the
    fp32 roundings of the partials and of their sum, all relative to |dZ|^T . |A|"""
    M, N = dZ.shape
    S, _ = split(M, N, A.shape[1], sms)
    mag = np.abs(dZ.astype(np.float64)).T @ np.abs(A.astype(np.float64))
    return (2 * 2.0 ** -11 + 2.0 ** -22 + (S + 1) * 2.0 ** -24) * mag
