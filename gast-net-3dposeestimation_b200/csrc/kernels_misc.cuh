// Small kernels of the lifting path: collapsed theta/phi row dots, attention mix, shrink,
// and the parameter-preparation kernels (BN folding, adjacency softmax, weight packing).
#pragma once
#include "gast_common.cuh"

namespace gast {

// ---------------------------------------------------------------------------------------
// ab[row][q] = X[row,:] . U[q,:] + cab[q],  q < Q (= 2*heads <= 8).   Warp per row.
// The theta/phi 1x1 convs followed by the concat-project conv (global_attention.py:60-72)
// collapse to these 2 dot products per head: f[i,j] = a_i + b_j.
// ---------------------------------------------------------------------------------------
template <int Q, typename T>
__global__ void rowdot_kernel(const T* __restrict__ X, int ldx, const float* __restrict__ U,
                              const float* __restrict__ cab, float* __restrict__ ab,
                              long long rows, int K) {
  long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const T* xr = X + row * ldx;
  float acc[Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) acc[q] = 0.f;
  for (int k = lane * 4; k < K; k += 128) {
    float4 xv = ld4(xr + k);
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      float4 u = ldg4(U + (long long)q * K + k);
      acc[q] = fmaf(xv.x, u.x, fmaf(xv.y, u.y, fmaf(xv.z, u.z, fmaf(xv.w, u.w, acc[q]))));
    }
  }
#pragma unroll
  for (int q = 0; q < Q; ++q) acc[q] = warp_sum(acc[q]);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < Q; ++q) ab[row * Q + q] = acc[q] + __ldg(cab + q);
  }
}

// Q = 8 (4 heads) version: U staged in shared memory, a warp walks rows with a grid stride, and the
// 8 partial sums are reduced with a halving butterfly (9 shuffles instead of 40).
template <typename T>
__global__ void rowdot8_kernel(const T* __restrict__ X, int ldx, const float* __restrict__ U,
                               const float* __restrict__ cab, float* __restrict__ ab, long long rows, int K) {
  extern __shared__ __align__(16) float us[];          // [8][K]
  for (int i = threadIdx.x * 4; i < 8 * K; i += blockDim.x * 4)
    *reinterpret_cast<float4*>(us + i) = ldg4(U + i);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const int sel = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);   // q owned after the butterfly
  const float cq = __ldg(cab + sel);
  // two rows per iteration: both rows' loads are in flight before the first FMA (one 512-byte request per
  // warp at a time left the kernel at 2.2 TB/s)
  for (long long row0 = warp; row0 < rows; row0 += 2 * nwarps) {
    const long long row1 = row0 + nwarps;
    const bool has1 = row1 < rows;
    const T* xr0 = X + row0 * ldx;
    const T* xr1 = X + (has1 ? row1 : row0) * ldx;
    float va[8], vb[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) { va[q] = 0.f; vb[q] = 0.f; }
    for (int k = lane * 4; k < K; k += 128) {
      const float4 xa = ld4(xr0 + k);
      const float4 xb = ld4(xr1 + k);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 u = *reinterpret_cast<const float4*>(us + q * K + k);
        va[q] = fmaf(xa.x, u.x, fmaf(xa.y, u.y, fmaf(xa.z, u.z, fmaf(xa.w, u.w, va[q]))));
        vb[q] = fmaf(xb.x, u.x, fmaf(xb.y, u.y, fmaf(xb.z, u.z, fmaf(xb.w, u.w, vb[q]))));
      }
    }
    const bool hi16 = lane & 16, hi8 = lane & 8, hi4 = lane & 4;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float* v = r ? vb : va;
      // halving butterfly: after the xor-16 step a lane keeps 4 of the 8 sums, then 2, then 1
      float w4[4], w2[2], w1;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float keep = hi16 ? v[i + 4] : v[i], send = hi16 ? v[i] : v[i + 4];
        w4[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float keep = hi8 ? w4[i + 2] : w4[i], send = hi8 ? w4[i] : w4[i + 2];
        w2[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
      }
      {
        const float keep = hi4 ? w2[1] : w2[0], send = hi4 ? w2[0] : w2[1];
        w1 = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
      w1 += __shfl_xor_sync(0xffffffffu, w1, 2);
      w1 += __shfl_xor_sync(0xffffffffu, w1, 1);
      if ((lane & 3) == 0 && (r == 0 || has1)) ab[(r ? row1 : row0) * 8 + sel] = w1 + cq;
    }
  }
}

// shrink (gast_net.py:60,99): y[row][o] = X[row,:] . Ws[o,:], o < 3.   Warp per row.  T, Y: the types of X and y
// (float, or __half: both in a half forward, X only at the fp16 precision)
template <typename T, typename Y>
__global__ void shrink_kernel(const T* __restrict__ X, int ldx, const float* __restrict__ Ws,
                              Y* __restrict__ y, long long rows, int K) {
  long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (row >= rows) return;
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
  if (lane == 0) { st1(y + row * 3, a0); st1(y + row * 3 + 1, a1); st1(y + row * 3 + 2, a2); }
}

// ---------------------------------------------------------------------------------------
// Test-time augmentation on the device (SURVEY.md §8f N1): the caller-side steps either side of
// the forward in reconstruction.evaluate / main.evaluate.
// ---------------------------------------------------------------------------------------
struct JointPerm { unsigned char p[32]; };   // left<->right partner of every joint (identity elsewhere)

// UnchunkedGenerator.next_epoch with augment=True (common/generators.py:210-233):
// out[0] = edge-padded sequence, out[1] = its mirrored twin (x *= -1, left/right keypoints swapped)
__global__ void tta_prepare_kernel(const float* __restrict__ seq, float* __restrict__ out, int T, int J, int F,
                                   int pad_l, int pad_r, JointPerm perm) {
  const int Tp = T + pad_l + pad_r;
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)Tp * J * F;
  if (idx >= n) return;
  int c = (int)(idx % F);
  int j = (int)((idx / F) % J);
  int t = (int)(idx / ((long long)F * J));
  int ts = min(max(t - pad_l, 0), T - 1);
  out[idx] = seq[((long long)ts * J + j) * F + c];
  float v = seq[((long long)ts * J + perm.p[j]) * F + c];
  out[n + idx] = (c == 0) ? -v : v;
}

// un-flip + average (main.py:314-318, reconstruction.py:163-167): out = mean(pred[0], unflip(pred[1]))
__global__ void tta_merge_kernel(const float* __restrict__ pred, float* __restrict__ out, int T, int J,
                                 JointPerm perm) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long n = (long long)T * J * 3;
  if (idx >= n) return;
  int c = (int)(idx % 3);
  int j = (int)((idx / 3) % J);
  long long t = idx / (3LL * J);
  float b = pred[n + (t * J + perm.p[j]) * 3 + c];
  if (c == 0) b = -b;
  out[idx] = (pred[idx] + b) / 2.0f;
}

// ---------------------------------------------------------------------------------------
// parameter preparation (eval mode)
// ---------------------------------------------------------------------------------------
// Attention mix of MultiGlobalGraph as its own kernel (global_attention.py:74-80):
//   Y[f, i, c] = sum_j att_h(c)[f, i, j] . G[f, j, c],   att_h = softmax_j(LeakyReLU_0.2(a_i + b_j)) + C_k
// Same arithmetic as the fused epilogue of the `g` GEMM, but at full occupancy: inside the GEMM only
// 8 warps per SM can work on it and the mix is latency-bound there (the epilogue warps stall on the softmax
// rows and the 17-term FMA chains while the tensor pipe idles).  One thread = (frame, 4 channels): the 17
// float4 of its channel group are read once (coalesced along the channel axis) and kept in registers, the
// attention rows of the block's frames are computed once into shared memory.  (A variant that requested the g values
// before the attention rows and staged a/b in shared memory measured 6-17 % slower: more registers live across the barrier.)
// ---------------------------------------------------------------------------------------
constexpr int MIX_THREADS = 128;
constexpr int MIX_JMAX = 20;
constexpr int MIX_JP = 20;        // padded row length of an attention row in shared memory (float4 reads)

// 17 float4 of g in registers per thread: 116 registers, 16 warps per SM.
template <typename T>
__global__ void __launch_bounds__(MIX_THREADS, 1)
global_mix_kernel(const T* __restrict__ G, int ldg, const float* __restrict__ ab, const float* __restrict__ ck,
                  T* __restrict__ Y, int ldy, long long F, int J, int heads, int Cg, int fpb) {
  extern __shared__ __align__(16) float att_s[];            // [fpb][heads][J][MIX_JP]
  const int tid = threadIdx.x;
  const int H2 = 2 * heads;
  const long long f0 = (long long)blockIdx.x * fpb;
  // ---- attention rows of this block's frames
  const int nrow = fpb * heads * J;
  for (int e = tid; e < nrow; e += MIX_THREADS) {
    const int i = e % J, h = (e / J) % heads, fs = e / (J * heads);
    const long long f = f0 + fs;
    float* dst = att_s + (size_t)e * MIX_JP;
    if (f < F) {
      const float* abf = ab + (f * J) * H2;
      const float a = __ldg(abf + i * H2 + 2 * h);
      float v[MIX_JMAX];
      float mx = -3.4e38f;
#pragma unroll
      for (int j = 0; j < MIX_JMAX; ++j)
        if (j < J) {
          float s = a + __ldg(abf + j * H2 + 2 * h + 1);
          s = (s >= 0.f) ? s : 0.2f * s;
          v[j] = s;
          mx = fmaxf(mx, s);
        }
      float sum = 0.f;
#pragma unroll
      for (int j = 0; j < MIX_JMAX; ++j)
        if (j < J) { v[j] = expf(v[j] - mx); sum += v[j]; }
      const float inv = 1.f / sum;
      const float* ckr = ck + ((long long)h * J + i) * J;
#pragma unroll
      for (int j = 0; j < MIX_JMAX; ++j) dst[j] = (j < J) ? v[j] * inv + __ldg(ckr + j) : 0.f;
    } else {
#pragma unroll
      for (int j = 0; j < MIX_JMAX; ++j) dst[j] = 0.f;
    }
  }
  __syncthreads();
  // ---- mix: thread = (frame slot, group of 4 channels)
  const int GV = (heads * Cg) / 4;
  for (int w = tid; w < fpb * GV; w += MIX_THREADS) {
    const int fs = w / GV, c = (w - fs * GV) * 4;
    const long long f = f0 + fs;
    if (f >= F) continue;
    const int h = c / Cg;
    float4 g[MIX_JMAX];
    const T* gp = G + (f * J) * (long long)ldg + c;
#pragma unroll
    for (int j = 0; j < MIX_JMAX; ++j)
      if (j < J) g[j] = ld4(gp + (long long)j * ldg);
    const float* arow = att_s + (size_t)((fs * heads + h) * J) * MIX_JP;
    T* yp = Y + (f * J) * (long long)ldy + c;
    for (int i = 0; i < J; ++i) {
      float a[MIX_JMAX];
#pragma unroll
      for (int q = 0; q < MIX_JMAX / 4; ++q) {
        const float4 t = *reinterpret_cast<const float4*>(arow + i * MIX_JP + q * 4);
        a[q * 4] = t.x; a[q * 4 + 1] = t.y; a[q * 4 + 2] = t.z; a[q * 4 + 3] = t.w;
      }
      float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int j = 0; j < MIX_JMAX; ++j)
        if (j < J) {
          o.x = fmaf(a[j], g[j].x, o.x); o.y = fmaf(a[j], g[j].y, o.y);
          o.z = fmaf(a[j], g[j].z, o.z); o.w = fmaf(a[j], g[j].w, o.w);
        }
      st4(yp + (long long)i * ldy, o);
    }
  }
}

// ---------------------------------------------------------------------------------------
struct BnP {  // eval BatchNorm as y = x*scale + shift ; null weight => identity
  const float* w; const float* b; const float* rm; const float* rv;
};

// out[n][kk*Cin + c] = w[n][c][kk] * scale(n);  bias_out[n] = shift(n)
__global__ void fold_conv_kernel(float* __restrict__ out, float* __restrict__ bias_out,
                                 const float* __restrict__ w, int N, int Cin, int taps, BnP bn) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)N * Cin * taps;
  if (idx < total) {
    int n = (int)(idx / ((long long)Cin * taps));
    int rem = (int)(idx - (long long)n * Cin * taps);
    int kk = rem / Cin, c = rem - kk * Cin;
    float s = bn.w ? bn.w[n] / sqrtf(bn.rv[n] + BN_EPS) : 1.f;
    out[idx] = w[((long long)n * Cin + c) * taps + kk] * s;
  }
  if (idx < N && bias_out) {
    int n = (int)idx;
    float s = bn.w ? bn.w[n] / sqrtf(bn.rv[n] + BN_EPS) : 1.f;
    bias_out[n] = bn.w ? (bn.b[n] - bn.rm[n] * s) : 0.f;
  }
}

// coef[z][c] = softmax over the nonzeros z of row i of e[c][.]  (x BN scale);
// the -9e15 fill of the reference (local_attention.py:40-42) makes masked entries exactly 0.
__global__ void semch_coef_kernel(float* __restrict__ coef, float* __restrict__ shift,
                                  const float* __restrict__ e, int e_row_stride, NbrTable nb,
                                  int nnz, int C, int J, BnP bn, const float* __restrict__ bias) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= C * J) return;
  int c = idx / J, i = idx - c * J;
  const float* er = e + (long long)c * e_row_stride;
  float s = bn.w ? bn.w[c] / sqrtf(bn.rv[c] + BN_EPS) : 1.f;
  int z0 = nb.row_ptr[i], z1 = nb.row_ptr[i + 1];
  float mx = -3.4e38f;
  for (int z = z0; z < z1; ++z) mx = fmaxf(mx, er[z]);
  float sum = 0.f;
  for (int z = z0; z < z1; ++z) sum += expf(er[z] - mx);
  for (int z = z0; z < z1; ++z) coef[(long long)z * C + c] = expf(er[z] - mx) / sum * s;
  if (i == 0 && shift) shift[c] = bn.w ? (bn.b[c] - bn.rm[c] * s) : (bias ? bias[c] : 0.f);
}

// packed[((tile)*128 + w*64 + cc)][k] = W[w][k][tile*64+cc]  (0 beyond Cout)
__global__ void semch_pack_kernel(float* __restrict__ packed, const float* __restrict__ W,
                                  int tiles, int Cin, int Cout) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)tiles * 128 * Cin;
  if (idx >= total) return;
  int k = (int)(idx % Cin);
  int n = (int)(idx / Cin);
  int tile = n >> 7, within = n & 127;
  int w = within >> 6, cc = within & 63;
  int c = tile * 64 + cc;
  packed[idx] = (c < Cout) ? W[((long long)w * Cin + k) * Cout + c] : 0.f;
}

// U[2h][k] = sum_m wc[m] theta_w[m][k];  U[2h+1][k] = sum_m wc[Ci+m] phi_w[m][k]
// cab[2h] = sum_m wc[m] theta_b[m];      cab[2h+1] = sum_m wc[Ci+m] phi_b[m]
__global__ void global_collapse_kernel(float* __restrict__ U, float* __restrict__ cab,
                                       const float* __restrict__ tw, const float* __restrict__ tb,
                                       const float* __restrict__ pw, const float* __restrict__ pb,
                                       const float* __restrict__ wc, int h, int C, int Ci) {
  // block = 32 input channels k (coalesced) x 8 slices of the inter-channel index m, reduced through shared memory
  // (one thread per k summing all Ci terms took 35-50 us per head: it runs in every training forward)
  __shared__ float sa[8][33], sb[8][33];
  const int kx = threadIdx.x & 31, mg = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + kx;
  float a = 0.f, b = 0.f;
  if (k < C)
    for (int m = mg; m < Ci; m += 8) {
      a = fmaf(wc[m], tw[(long long)m * C + k], a);
      b = fmaf(wc[Ci + m], pw[(long long)m * C + k], b);
    }
  sa[mg][kx] = a; sb[mg][kx] = b;
  __syncthreads();
  if (mg == 0 && k < C) {
    float ra = 0.f, rb = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { ra += sa[i][kx]; rb += sb[i][kx]; }
    U[(long long)(2 * h) * C + k] = ra;
    U[(long long)(2 * h + 1) * C + k] = rb;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float ca = 0.f, cb = 0.f;
    for (int m = 0; m < Ci; ++m) { ca = fmaf(wc[m], tb[m], ca); cb = fmaf(wc[Ci + m], pb[m], cb); }
    cab[2 * h] = ca;
    cab[2 * h + 1] = cb;
  }
}

// We[kk*Fin+i][c] = w[c][i][kk] * s_in[i] * s_e[c];  be[c] = s_e[c]*sum w*t_in + t_e[c]
__global__ void expand_fold_kernel(float* __restrict__ We, float* __restrict__ be,
                                   const float* __restrict__ w, int C, int Fin, int taps,
                                   BnP bin, BnP bex) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float se = bex.w[c] / sqrtf(bex.rv[c] + BN_EPS);
  float te = bex.b[c] - bex.rm[c] * se;
  float acc = 0.f;
  for (int kk = 0; kk < taps; ++kk)
    for (int i = 0; i < Fin; ++i) {
      float si = bin.w[i] / sqrtf(bin.rv[i] + BN_EPS);
      float ti = bin.b[i] - bin.rm[i] * si;
      float wv = w[((long long)c * Fin + i) * taps + kk];
      We[(long long)(kk * Fin + i) * C + c] = wv * si * se;   // [k][C]: the expand kernel reads a float4 of 4 channels per k
      acc = fmaf(wv, ti, acc);
    }
  be[c] = se * acc + te;
}

}  // namespace gast
