// HBM-bound kernels of the lifting path: the expand stage staged through shared memory (every width, the forward and the
// streaming push) and the shrink layer with mpjpe in its epilogue (gast_forward_mpjpe).
//
// Measured (on the earlier B200 build) and NOT kept: persistent bulk-copy
// (cp.async.bulk + mbarrier ring) forms of the attention mix -- register-resident g and g kept in shared memory with
// 4 channels x 3-4 output joints per thread -- and of the theta/phi row dots (one pipeline per warp).  The mix variants
// were 0-40 % slower than global_mix_kernel, the row dots equal to rowdot8_kernel: both kernels are bound by their own
// dependent instruction chains (softmax rows, 17-term FMA chains, butterfly reductions), not by how the bytes arrive.
#pragma once
#include "gast_common.cuh"
#include "kernels_misc.cuh"

namespace gast {

// ---------------------------------------------------------------------------------------
// expand stage (gast_net.py:163-164): ReLU(BN(Conv_{(k,1), F->C}(BN_in(x)))) with both BNs folded into We/be.
// x: (B,T,J,Fin) ; out: (rows = B*T0*J, C).  A block owns EXS_ROWS consecutive output rows.  Their taps*Fin input
// values are gathered ONCE into shared memory (a first version had every one of the C/4 threads of a row request them
// again through L1: 48 loads in flight per thread, 126 registers, 16 warps per SM, 1.7 TB/s of output); a thread then
// keeps the folded weights of its 4 channels in registers and walks the block's rows: 2 broadcast shared-memory reads,
// 4*KF FMAs (bias first, then k ascending) and one coalesced 16-byte store per row, full occupancy.
// A block covers at most EXS_CHUNK channels; wider layers take more chunks along blockIdx.y, each staging the same rows.
// ---------------------------------------------------------------------------------------
constexpr int EXS_ROWS = 128;
constexpr int EXS_THREADS = 256;
constexpr int EXS_CHUNK = 4 * EXS_THREADS;               // channels per block: 4 per thread
constexpr int EXP_MAXKF = 10;   // taps * in_features supported by the register path (3*2 = 6; 5*2 = 10)
// In, Out: the types of x and out (float, or __half: both in a half forward, out only at the fp16 precision)
template <int KFT, typename In, typename Out>   // register-resident K = taps * in_features rounded up: 6 or EXP_MAXKF
__global__ void __launch_bounds__(EXS_THREADS)
expand_rows_kernel(const In* __restrict__ x, const float* __restrict__ We, const float* __restrict__ be,
                   Out* __restrict__ out, long long rows, int J, int T, int T0, int stride, int taps, int Fin, int C) {
  constexpr int KP = (KFT + 3) & ~3;                      // padded row of staged inputs (float4 reads)
  __shared__ __align__(16) float xs[EXS_ROWS * KP];
  const int tid = threadIdx.x;
  const int KF = taps * Fin;
  const long long r0 = (long long)blockIdx.x * EXS_ROWS;
  const int nrows = (int)((rows - r0 < EXS_ROWS) ? (rows - r0) : EXS_ROWS);
  for (int e = tid; e < EXS_ROWS * KP; e += EXS_THREADS) {
    const int rr = e / KP, k = e - rr * KP;
    float v = 0.f;
    if (rr < nrows && k < KF) {
      const int row = (int)(r0 + rr);                     // the host checks rows < 2^31
      const int f = row / J, j = row - f * J;
      const int b = f / T0, t = f - b * T0;
      const int kk = k / Fin, i = k - kk * Fin;
      v = ld1(x + (((long long)b * T + (long long)t * stride + kk) * J + j) * Fin + i);
    }
    xs[e] = v;
  }
  const int c0 = blockIdx.y * EXS_CHUNK;                  // first channel of this block's chunk
  const int cq = min(C - c0, EXS_CHUNK) >> 2;             // channel groups (threads) per row
  const int rpp = EXS_THREADS / cq;                       // rows per pass of the block
  const int cg = tid % cq, rsub = tid / cq;
  const int c = c0 + cg * 4;
  float w[4][KFT];
#pragma unroll
  for (int k = 0; k < KFT; ++k) {
    float4 wk = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < KF) wk = ldg4(We + (long long)k * C + c);
    w[0][k] = wk.x; w[1][k] = wk.y; w[2][k] = wk.z; w[3][k] = wk.w;
  }
  const float4 b4 = ldg4(be + c);
  __syncthreads();
  if (rsub >= rpp) return;                                // (256 % cq != 0: the surplus threads have no row)
  Out* op = out + (r0 + rsub) * C + c;
  const long long ostep = (long long)rpp * C;
#pragma unroll 4
  for (int rr = rsub; rr < nrows; rr += rpp, op += ostep) {
    float xv[KP];
#pragma unroll
    for (int q = 0; q < KP / 4; ++q) {
      const float4 t4 = *reinterpret_cast<const float4*>(xs + rr * KP + q * 4);
      xv[q * 4] = t4.x; xv[q * 4 + 1] = t4.y; xv[q * 4 + 2] = t4.z; xv[q * 4 + 3] = t4.w;
    }
    float v0 = b4.x, v1 = b4.y, v2 = b4.z, v3 = b4.w;
#pragma unroll
    for (int k = 0; k < KFT; ++k) {
      v0 = fmaf(w[0][k], xv[k], v0); v1 = fmaf(w[1][k], xv[k], v1);
      v2 = fmaf(w[2][k], xv[k], v2); v3 = fmaf(w[3][k], xv[k], v3);
    }
    st4(op, make_float4(fmaxf(v0, 0.f), fmaxf(v1, 0.f), fmaxf(v2, 0.f), fmaxf(v3, 0.f)));
  }
}

// ---------------------------------------------------------------------------------------
// shrink (gast_net.py:60,99) with mpjpe (common/loss.py:5-11) in its epilogue: the warp that produced the 3 coordinates
// of an output joint also takes ||y - target|| of it.  Partial sums are double (like mpjpe_kernel); the last block to
// finish (atomic ticket) adds the block partials in index order, so the loss does not depend on the scheduling, and
// resets the ticket for the next call (CUDA-graph replay safe).  y is written as by shrink_kernel (same FMA order).
// X: float, or __half at the fp16 precision (y, target and the loss stay float).
// ---------------------------------------------------------------------------------------
constexpr int SHL_MAXBLOCKS = 1024;
template <typename T>
__global__ void __launch_bounds__(256)
shrink_mpjpe_kernel(const T* __restrict__ X, int ldx, const float* __restrict__ Ws, float* __restrict__ y,
                    long long rows, int K, const float* __restrict__ target, double* __restrict__ partial,
                    unsigned* __restrict__ ticket, float* __restrict__ loss) {
  const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
  const long long nw = (long long)gridDim.x * 8;
  double acc = 0.0;
  for (long long row = (long long)blockIdx.x * 8 + wrp; row < rows; row += nw) {
    const T* xr = X + row * ldx;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int k = lane * 4; k < K; k += 128) {
      float4 xv = ld4(xr + k);
      float4 w0 = ldg4(Ws + k), w1 = ldg4(Ws + K + k), w2 = ldg4(Ws + 2 * K + k);
      a0 = fmaf(xv.x, w0.x, fmaf(xv.y, w0.y, fmaf(xv.z, w0.z, fmaf(xv.w, w0.w, a0))));
      a1 = fmaf(xv.x, w1.x, fmaf(xv.y, w1.y, fmaf(xv.z, w1.z, fmaf(xv.w, w1.w, a1))));
      a2 = fmaf(xv.x, w2.x, fmaf(xv.y, w2.y, fmaf(xv.z, w2.z, fmaf(xv.w, w2.w, a2))));
    }
    a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2);
    if (lane == 0) {
      y[row * 3 + 0] = a0; y[row * 3 + 1] = a1; y[row * 3 + 2] = a2;
      const float d0 = a0 - target[row * 3], d1 = a1 - target[row * 3 + 1], d2 = a2 - target[row * 3 + 2];
      acc += (double)sqrtf(fmaf(d2, d2, fmaf(d1, d1, d0 * d0)));       // same expression as mpjpe_kernel (D = 3)
    }
  }
  __shared__ double sh[8];
  __shared__ bool last;
  if (lane == 0) sh[wrp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int i = 0; i < 8; ++i) v += sh[i];
    partial[blockIdx.x] = v;
    __threadfence();
    last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (threadIdx.x < 32) {
    double v = 0.0;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += 32) v += __ldcg(partial + i);
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) { *loss = (float)(v / (double)rows); *ticket = 0u; }
  }
}

}  // namespace gast
