// Training-mode kernels of the lifting path (row a12 of SURVEY.md §8): batch-statistics BatchNorm
// forward/backward, the joint-mixing operators and their adjoints, gather/scatter of the temporal
// taps, and small reductions.  The training batch of the reference is small (b=128: 19,584 /
// 6,528 / 2,176 rows per stage), so these kernels are written for exactness and simplicity; the
// dense contractions (Z = A.W^T, dA = dZ.W, dW = dZ^T.A) run on the same GEMM kernels as inference.
#pragma once
#include "gast_common.cuh"

namespace gast {

// ----------------------------------------------------------------------------------------------
// column reductions over rows:  out[n] (+)= sum_m f(...)    (block = 32 columns x 8 row lanes)
// ----------------------------------------------------------------------------------------------
// sum and sum of squares per column, accumulated in double (BatchNorm batch statistics,
// nn.BatchNorm2d training mode: gast_net.py:20,58-59,147,149 and the attention modules)
__global__ void col_stats_kernel(const float* __restrict__ Z, long long M, int N, int ld,
                                 double* __restrict__ sum, double* __restrict__ sumsq) {
  const int n = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;                 // 0..7
  double s = 0.0, q = 0.0;
  if (n < N) {
    for (long long m = (long long)blockIdx.y * 8 + rl; m < M; m += (long long)gridDim.y * 8) {
      double v = (double)Z[m * ld + n];
      s += v; q += v * v;
    }
  }
  __shared__ double sh[2][8][33];
  sh[0][rl][threadIdx.x & 31] = s;
  sh[1][rl][threadIdx.x & 31] = q;
  __syncthreads();
  if (rl == 0 && n < N) {
    for (int i = 1; i < 8; ++i) { s += sh[0][i][threadIdx.x & 31]; q += sh[1][i][threadIdx.x & 31]; }
    atomicAdd(sum + n, s);
    atomicAdd(sumsq + n, q);
  }
}

// mean / invstd from the sums; running statistics updated like torch (momentum 0.1, unbiased var)
__global__ void bn_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ sumsq, long long M,
                                   int N, float* __restrict__ mean, float* __restrict__ invstd,
                                   float* __restrict__ running_mean, float* __restrict__ running_var,
                                   float momentum) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  double mu = sum[n] / (double)M;
  double var = sumsq[n] / (double)M - mu * mu;
  if (var < 0) var = 0;
  mean[n] = (float)mu;
  invstd[n] = (float)(1.0 / sqrt(var + (double)BN_EPS));
  if (running_mean) {
    double unb = (M > 1) ? var * (double)M / (double)(M - 1) : var;
    running_mean[n] = (1.f - momentum) * running_mean[n] + momentum * (float)mu;
    running_var[n] = (1.f - momentum) * running_var[n] + momentum * (float)unb;
  }
}

// frozen (eval-mode) BatchNorm: mean / invstd from the running statistics, which are only read
__global__ void bn_running_kernel(const float* __restrict__ running_mean, const float* __restrict__ running_var, int N,
                                  float* __restrict__ mean, float* __restrict__ invstd) {
  int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  mean[n] = running_mean[n];
  invstd[n] = (float)(1.0 / sqrt((double)running_var[n] + (double)BN_EPS));
}

// Y = [res +] drop( relu( (Z-mean)*invstd*gamma + beta ) )      (relu / res / drop optional)
// res rows follow a frame map (residual slice of the temporal stage, gast_net.py:243)
__global__ void bn_apply_kernel(const float* __restrict__ Z, int ldz, const float* __restrict__ mean,
                                const float* __restrict__ invstd, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int relu, const float* __restrict__ res, int ldres,
                                RowMap rmap, int J, const unsigned char* __restrict__ keep, float keep_scale,
                                float* __restrict__ Y, int ldy, long long M, int N) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * N) return;
  long long m = idx / N;
  int n = (int)(idx - m * N);
  float v = (Z[m * ldz + n] - mean[n]) * invstd[n] * gamma[n] + beta[n];
  if (relu) v = fmaxf(v, 0.f);
  if (keep) v = keep[idx] ? v * keep_scale : 0.f;
  if (res) {
    long long f = m / J;
    int j = (int)(m - f * J);
    v += res[(map_frame(rmap, f) * J + j) * ldres + n];
  }
  Y[m * ldy + n] = v;
}

// dgamma[n] = sum_m dYhat*xhat ; dbeta[n] = sum_m dYhat,   dYhat = dY * keep * [bn(Z) > 0 if relu]
__global__ void bn_bwd_reduce_kernel(const float* __restrict__ dY, int lddy, const float* __restrict__ Z, int ldz,
                                     const float* __restrict__ mean, const float* __restrict__ invstd,
                                     const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
                                     const unsigned char* __restrict__ keep, float keep_scale, long long M, int N,
                                     double* __restrict__ dgamma, double* __restrict__ dbeta) {
  const int n = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  double g = 0.0, b = 0.0;
  if (n < N) {
    const float mu = mean[n], is = invstd[n], ga = gamma[n], be = beta[n];
    for (long long m = (long long)blockIdx.y * 8 + rl; m < M; m += (long long)gridDim.y * 8) {
      float xh = (Z[m * ldz + n] - mu) * is;
      float d = dY[m * lddy + n];
      if (keep) d = keep[m * N + n] ? d * keep_scale : 0.f;
      if (relu && !(xh * ga + be > 0.f)) d = 0.f;
      g += (double)d * xh;
      b += (double)d;
    }
  }
  __shared__ double sh[2][8][33];
  sh[0][rl][threadIdx.x & 31] = g;
  sh[1][rl][threadIdx.x & 31] = b;
  __syncthreads();
  if (rl == 0 && n < N) {
    for (int i = 1; i < 8; ++i) { g += sh[0][i][threadIdx.x & 31]; b += sh[1][i][threadIdx.x & 31]; }
    atomicAdd(dgamma + n, g);
    atomicAdd(dbeta + n, b);
  }
}

// dZ = gamma*invstd*(dYhat - dbeta/M - xhat*dgamma/M); also writes the float parameter grads (when g_gamma / g_beta are
// given).  FROZEN (running statistics, eval mode): mean / invstd do not depend on Z, so dZ = gamma*invstd*dYhat, and
// dgamma / dbeta are read only for the parameter grads (null in an input-only backward).
template <bool FROZEN>
__global__ void bn_bwd_apply_kernel(const float* __restrict__ dY, int lddy, const float* __restrict__ Z, int ldz,
                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                    const float* __restrict__ gamma, const float* __restrict__ beta, int relu,
                                    const unsigned char* __restrict__ keep, float keep_scale, long long M, int N,
                                    const double* __restrict__ dgamma, const double* __restrict__ dbeta,
                                    float* __restrict__ dZ, int lddz, float* __restrict__ g_gamma,
                                    float* __restrict__ g_beta) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * N) return;
  long long m = idx / N;
  int n = (int)(idx - m * N);
  const float is = invstd[n], ga = gamma[n];
  float xh = (Z[m * ldz + n] - mean[n]) * is;
  float d = dY[m * lddy + n];
  if (keep) d = keep[idx] ? d * keep_scale : 0.f;
  if (relu && !(xh * ga + beta[n] > 0.f)) d = 0.f;
  if (FROZEN) {
    dZ[m * lddz + n] = ga * is * d;
  } else {
    const float invM = 1.f / (float)M;
    dZ[m * lddz + n] = ga * is * (d - (float)dbeta[n] * invM - xh * (float)dgamma[n] * invM);
  }
  if (m == 0) {
    if (g_gamma) g_gamma[n] = (float)dgamma[n];
    if (g_beta) g_beta[n] = (float)dbeta[n];
  }
}

// out[n] = sum_m X[m][n]   (bias gradients)
__global__ void col_sum_kernel(const float* __restrict__ X, long long M, int N, int ld, double* __restrict__ out) {
  const int n = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  double s = 0.0;
  if (n < N)
    for (long long m = (long long)blockIdx.y * 8 + rl; m < M; m += (long long)gridDim.y * 8) s += (double)X[m * ld + n];
  __shared__ double sh[8][33];
  sh[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && n < N) {
    for (int i = 1; i < 8; ++i) s += sh[i][threadIdx.x & 31];
    atomicAdd(out + n, s);
  }
}

__global__ void d2f_kernel(const double* __restrict__ in, float* __restrict__ out, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (float)in[i];
}

// ----------------------------------------------------------------------------------------------
// layout helpers
// ----------------------------------------------------------------------------------------------
// Weight gradient  dW[N][K] = dZ[M][N]^T . A[M][K]  ("TN" GEMM: the contraction runs over the ROWS of both
// operands, so both tiles are read in their natural row-major form -- no transposed copies).  The training batch
// makes M the only large dimension (b=128: M = 19,584 rows against N x K = 256 x 384), so the work is split over
// M: grid = (N tiles, K tiles, S row ranges); split s writes its partial [N][K] product to part + s*N*K and
// wgrad_reduce_kernel sums the S partials in a fixed order (deterministic, unlike atomics).
// 128 x 128 tile, 256 threads, 8 x 8 micro-tiles as 2 x 2 blocks of 4 x 4 (conflict-free 128-bit smem reads),
// rows staged 16 at a time with register prefetch.  Exact fp32 (FFMA).
constexpr int WG_T = 128, WG_M = 16;
__global__ void __launch_bounds__(256)
wgrad_tn_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ A, int lda, long long M, int N, int K,
                long long rows_per_split, float* __restrict__ part) {
  __shared__ __align__(16) float sZ[2][WG_M][WG_T];
  __shared__ __align__(16) float sA[2][WG_M][WG_T];
  const int n0 = blockIdx.x * WG_T, k0 = blockIdx.y * WG_T;
  const long long m_beg = (long long)blockIdx.z * rows_per_split;
  const long long m_end = min(M, m_beg + rows_per_split);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  // loader: thread -> (row lr of the 16-row slab, 16-byte column group lc): 16 rows x 32 float4 = 512 float4 per
  // operand, 2 per thread
  const int lr = tid >> 5, lc = (tid & 31) * 4;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const bool vecZ = (lddz % 4 == 0) && ((reinterpret_cast<uintptr_t>(dZ) & 15) == 0);
  const bool vecA = (lda % 4 == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  auto load4 = [&](const float* base, int ld, long long m, int c, int lim, bool vec) -> float4 {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < m_end) {
      const float* p = base + m * ld + c;
      if (vec && c + 3 < lim) v = ldg4(p);
      else {
        if (c < lim) v.x = __ldg(p);
        if (c + 1 < lim) v.y = __ldg(p + 1);
        if (c + 2 < lim) v.z = __ldg(p + 2);
        if (c + 3 < lim) v.w = __ldg(p + 3);
      }
    }
    return v;
  };
  float4 rz[2], ra[2];
  auto fetch = [&](long long m0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      rz[h] = load4(dZ, lddz, m0 + lr + 8 * h, n0 + lc, N, vecZ);
      ra[h] = load4(A, lda, m0 + lr + 8 * h, k0 + lc, K, vecA);
    }
  };
  auto stash = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      *reinterpret_cast<float4*>(&sZ[buf][lr + 8 * h][lc]) = rz[h];
      *reinterpret_cast<float4*>(&sA[buf][lr + 8 * h][lc]) = ra[h];
    }
  };
  int buf = 0;
  if (m_beg < m_end) {
    fetch(m_beg);
    stash(0);
  }
  __syncthreads();
  for (long long m0 = m_beg; m0 < m_end; m0 += WG_M) {
    const bool more = m0 + WG_M < m_end;
    if (more) fetch(m0 + WG_M);
#pragma unroll
    for (int mm = 0; mm < WG_M; ++mm) {
      const float4 z0 = *reinterpret_cast<const float4*>(&sZ[buf][mm][ty * 4]);
      const float4 z1 = *reinterpret_cast<const float4*>(&sZ[buf][mm][64 + ty * 4]);
      const float4 a0 = *reinterpret_cast<const float4*>(&sA[buf][mm][tx * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&sA[buf][mm][64 + tx * 4]);
      const float zv[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(zv[i], av[j], acc[i][j]);
    }
    if (more) stash(buf ^ 1);
    __syncthreads();
    buf ^= 1;
  }
  float* out = part + (long long)blockIdx.z * N * K;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int n = n0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (n >= N) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int k = k0 + jh * 64 + tx * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (k + j < K) out[(long long)n * K + k + j] = acc[i][jh * 4 + j];
    }
  }
}

// dW[n][k] (leading dim lddw) = sum over the S partial products, in split order
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int S, int N, int K, float* __restrict__ dW, int lddw) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long NK = (long long)N * K;
  if (idx >= NK) return;
  float s = 0.f;
  for (int i = 0; i < S; ++i) s += part[(long long)i * NK + idx];
  const int n = (int)(idx / K);
  dW[(long long)n * lddw + (idx - (long long)n * K)] = s;
}

// ----------------------------------------------------------------------------------------------
// out[c][r] = in[r][c]   (in: R x C with leading dim ldi; out: C x ldo, columns r >= R zero-filled by memset)
__global__ void transpose_kernel(const float* __restrict__ in, long long R, int C, int ldi, float* __restrict__ out,
                                 long long ldo) {
  __shared__ float t[32][33];
  long long r0 = (long long)blockIdx.x * 32;
  int c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += 8) {
    long long r = r0 + i;
    int c = c0 + threadIdx.x;
    t[i][threadIdx.x] = (r < R && c < C) ? in[r * ldi + c] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += 8) {
    int c = c0 + i;
    long long r = r0 + threadIdx.x;
    if (c < C && r < R) out[(long long)c * ldo + r] = t[threadIdx.x][i];
  }
}

// Gather a (possibly tapped / frame-mapped) A segment into a dense matrix:  dst[m][coff + k] = seg(m, k)
__global__ void seg_gather_kernel(ASeg sg, int J, long long F, float* __restrict__ dst, int ldd, int coff) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long M = F * J;
  if (idx >= M * sg.K) return;
  long long m = idx / sg.K;
  int k = (int)(idx - m * sg.K);
  long long f = m / J;
  int j = (int)(m - f * J);
  int tap = k / sg.Kc, c = k - tap * sg.Kc;
  dst[m * ldd + coff + k] = sg.base[(map_frame(sg.map, f) * J + j) * (long long)sg.ld + tap * sg.tap_stride + c];
}

// Adjoint of the gather:  grad_seg(m, k) += src[m][coff + k]   (atomic: taps / residuals may overlap)
__global__ void seg_scatter_add_kernel(ASeg sg, int J, long long F, const float* __restrict__ src, int lds, int coff) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long M = F * J;
  if (idx >= M * sg.K) return;
  long long m = idx / sg.K;
  int k = (int)(idx - m * sg.K);
  long long f = m / J;
  int j = (int)(m - f * J);
  int tap = k / sg.Kc, c = k - tap * sg.Kc;
  float* dstp = const_cast<float*>(sg.base) + (map_frame(sg.map, f) * J + j) * (long long)sg.ld + tap * sg.tap_stride + c;
  atomicAdd(dstp, src[m * lds + coff + k]);
}

// y[i] += x[i]
__global__ void add_inplace_kernel(float* __restrict__ y, const float* __restrict__ x, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] += x[i];
}

// generic strided copy: dst[m][n] = src[m][n]  (optionally accumulating)
__global__ void copy2d_kernel(const float* __restrict__ src, int lds, float* __restrict__ dst, int ldd, long long M,
                              int N, int accumulate) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * N) return;
  long long m = idx / N;
  int n = (int)(idx - m * N);
  float v = src[m * lds + n];
  if (accumulate) dst[m * ldd + n] += v; else dst[m * ldd + n] = v;
}

// counter-based dropout mask (nn.Dropout semantics: keep with prob 1-p, scale 1/(1-p)); the
// stream is ours, not torch's -- loss-match tests use p = 0 (SURVEY.md §7 "Dropout parity")
// `dseed` (device, may be null): added to the seed, so that a CUDA-graph replay of the step -- whose kernel arguments
// are frozen -- still draws a fresh mask (dropout_bump_kernel advances it once per forward).
__global__ void dropout_mask_kernel(unsigned char* __restrict__ keep, long long n, float p, unsigned long long seed,
                                    const unsigned long long* __restrict__ dseed) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (dseed) seed += *dseed;
  unsigned long long x = (unsigned long long)i * 0x9E3779B97F4A7C15ull + seed;
  x ^= x >> 30; x *= 0xBF58476D1CE4E5B9ull; x ^= x >> 27; x *= 0x94D049BB133111EBull; x ^= x >> 31;
  float u = (float)(x >> 40) * (1.0f / 16777216.0f);
  keep[i] = (u >= p) ? 1 : 0;
}

__global__ void dropout_bump_kernel(unsigned long long* dseed) { *dseed += 0xD1B54A32D192ED03ull; }

// ----------------------------------------------------------------------------------------------
// SemCH joint mixing and its adjoints (model/local_attention.py:35-53)
//   H: (M, 2C) = [X.W0 | X.W1] of one mask;  A: coef[z][c] = softmax over the row's nonzeros
//   S[i,c] = sum_z in row i  A[z,c] * H_{w}[ (f, col z), c ],  w = 0 if col z == i else 1
// ----------------------------------------------------------------------------------------------
__global__ void semch_mix_fwd_kernel(const float* __restrict__ H, int ldh, const float* __restrict__ coef, NbrTable nb,
                                     int J, long long F, int C, float* __restrict__ S, int lds) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long M = F * J;
  if (idx >= M * C) return;
  long long m = idx / C;
  int c = (int)(idx - m * C);
  long long f = m / J;
  int i = (int)(m - f * J);
  float s = 0.f;
  for (int z = nb.row_ptr[i]; z < nb.row_ptr[i + 1]; ++z) {
    int jn = nb.col[z];
    float h = H[(f * J + jn) * ldh + ((jn == i) ? 0 : C) + c];
    s = fmaf(coef[(long long)z * C + c], h, s);
  }
  S[m * lds + c] = s;
}

// dH0[i,c] = A[self(i),c] dS[i,c];  dH1[j,c] = sum_{z: col z = j, row z != j} A[z,c] dS[(f,row z),c]
// (rowof[z] = row of nonzero z, precomputed on the host)
struct NbrRows { unsigned char rowof[164]; };
__global__ void semch_mix_bwd_kernel(const float* __restrict__ dS, int lds, const float* __restrict__ coef, NbrTable nb,
                                     NbrRows nr, int nnz, int J, long long F, int C, float* __restrict__ dH, int ldh) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long M = F * J;
  if (idx >= M * C) return;
  long long m = idx / C;
  int c = (int)(idx - m * C);
  long long f = m / J;
  int j = (int)(m - f * J);
  float d0 = 0.f, d1 = 0.f;
  for (int z = 0; z < nnz; ++z) {
    if (nb.col[z] != j) continue;
    int i = nr.rowof[z];
    float a = coef[(long long)z * C + c] * dS[(f * J + i) * lds + c];
    if (i == j) d0 += a; else d1 += a;
  }
  dH[m * ldh + c] = d0;
  dH[m * ldh + C + c] = d1;
}

// dA[z][c] = sum_f dS[(f,row z),c] * H_w[(f,col z),c]     (thread per (z,c), loop over frames)
__global__ void semch_dcoef_kernel(const float* __restrict__ dS, int lds, const float* __restrict__ H, int ldh,
                                   NbrTable nb, NbrRows nr, int nnz, int J, long long F, int C,
                                   double* __restrict__ part /* [gridDim.y][nnz*C] */) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nnz * C) return;
  int z = idx / C, c = idx - z * C;
  int i = nr.rowof[z], jn = nb.col[z];
  int off = (jn == i) ? 0 : C;
  // frames split over gridDim.y (one thread per output summing every frame took 0.12 ms per mask at b = 128);
  // the partial sums are added in split order by semch_dcoef_reduce_kernel: deterministic
  const long long per = (F + gridDim.y - 1) / gridDim.y;
  const long long f0 = (long long)blockIdx.y * per, f1 = min(F, f0 + per);
  double s = 0.0;
  for (long long f = f0; f < f1; ++f)
    s += (double)dS[(f * J + i) * lds + c] * (double)H[(f * J + jn) * ldh + off + c];
  part[(long long)blockIdx.y * nnz * C + idx] = s;
}

__global__ void semch_dcoef_reduce_kernel(const double* __restrict__ part, int S, int n, float* __restrict__ dA) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  double s = 0.0;
  for (int i = 0; i < S; ++i) s += part[(long long)i * n + idx];
  dA[idx] = (float)s;
}

// softmax backward per (c,row):  de[c][z] = A[z,c] * (dA[z,c] - sum_{z' in row} A[z',c] dA[z',c])
__global__ void semch_de_kernel(const float* __restrict__ coef, const float* __restrict__ dA, NbrTable nb, int nnz,
                                int J, int C, float* __restrict__ de /* [C][nnz] */) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= C * J) return;
  int c = idx / J, i = idx - c * J;
  float dot = 0.f;
  for (int z = nb.row_ptr[i]; z < nb.row_ptr[i + 1]; ++z) dot += coef[(long long)z * C + c] * dA[(long long)z * C + c];
  for (int z = nb.row_ptr[i]; z < nb.row_ptr[i + 1]; ++z)
    de[(long long)c * nnz + z] = coef[(long long)z * C + c] * (dA[(long long)z * C + c] - dot);
}

// ----------------------------------------------------------------------------------------------
// global attention mixing and its adjoint (model/global_attention.py:52-82); one block per frame
//   G: (M, Ng) stacked heads (+bias),  ab: (M, 2H) with a_h(i), b_h(j),  Ck: (H, J, J)
//   P = softmax_j(LeakyReLU_0.2(a_i + b_j)),  att = P + Ck,  Y[i,:] = sum_j att[i,j] G[j,:]
// ----------------------------------------------------------------------------------------------
__global__ void att_mix_fwd_kernel(const float* __restrict__ G, int ldg, const float* __restrict__ ab,
                                   const float* __restrict__ ck, int J, int H, int Cg, float* __restrict__ Y, int ldy) {
  extern __shared__ float sm[];            // att[H][J][J]
  const long long f = blockIdx.x;
  const int H2 = 2 * H;
  for (int t = threadIdx.x; t < H * J; t += blockDim.x) {
    int h = t / J, i = t - h * J;
    float a = ab[(f * J + i) * H2 + 2 * h];
    float mx = -3.4e38f;
    float* row = sm + (h * J + i) * J;
    for (int j = 0; j < J; ++j) {
      float s = a + ab[(f * J + j) * H2 + 2 * h + 1];
      s = (s >= 0.f) ? s : 0.2f * s;
      row[j] = s; mx = fmaxf(mx, s);
    }
    float sum = 0.f;
    for (int j = 0; j < J; ++j) { float e = expf(row[j] - mx); row[j] = e; sum += e; }
    float inv = 1.f / sum;
    for (int j = 0; j < J; ++j) row[j] = row[j] * inv + ck[(h * J + i) * J + j];
  }
  __syncthreads();
  const int Ng = H * Cg;
  for (int t = threadIdx.x; t < J * Ng; t += blockDim.x) {
    int i = t / Ng, n = t - i * Ng;
    int h = n / Cg;
    const float* row = sm + (h * J + i) * J;
    float s = 0.f;
    for (int j = 0; j < J; ++j) s = fmaf(row[j], G[(f * J + j) * ldg + n], s);
    Y[(f * J + i) * ldy + n] = s;
  }
}

// out[n] = sum_m X[m][n] in a FIXED order (block = 32 columns x 8 row lanes, every lane walks its rows in order, the
// lanes are added in order): run-to-run reproducible, unlike atomics.  Used for dC_k: its float atomics were the only
// run-to-run difference of the whole training step (tools/train_determinism.py), and Adam(amsgrad) amplifies a 1e-8
// difference in one gradient into +-lr differences of 3-15 % of the parameters within three steps.
__global__ void col_sum_det_kernel(const float* __restrict__ X, long long M, int N, float* __restrict__ out) {
  __shared__ double sh[8][33];
  const int n = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rl = threadIdx.x >> 5;
  double s = 0.0;
  if (n < N)
    for (long long m = rl; m < M; m += 8) s += (double)X[m * N + n];
  sh[rl][threadIdx.x & 31] = s;
  __syncthreads();
  if (rl == 0 && n < N) {
    for (int i = 1; i < 8; ++i) s += sh[i][threadIdx.x & 31];
    out[n] = (float)s;
  }
}

// adjoint: dG, dab, and this frame's contribution to dCk (dCk_part[f][H*J*J], summed over the frames by col_sum_det_kernel)
__global__ void att_mix_bwd_kernel(const float* __restrict__ dY, int lddy, const float* __restrict__ G, int ldg,
                                   const float* __restrict__ ab, const float* __restrict__ ck, int J, int H, int Cg,
                                   float* __restrict__ dG, int lddg, float* __restrict__ dab,
                                   float* __restrict__ dCk_part) {
  extern __shared__ float sm[];            // P[H][J][J], att[H][J][J], datt[H][J][J], lin[H][J][J]
  const long long f = blockIdx.x;
  const int H2 = 2 * H, JJ = J * J;
  float* P = sm;
  float* att = sm + H * JJ;
  float* datt = sm + 2 * H * JJ;
  float* lin = sm + 3 * H * JJ;            // pre-activation a_i + b_j
  for (int t = threadIdx.x; t < H * J; t += blockDim.x) {
    int h = t / J, i = t - h * J;
    float a = ab[(f * J + i) * H2 + 2 * h];
    float mx = -3.4e38f;
    float* row = P + (h * J + i) * J;
    for (int j = 0; j < J; ++j) {
      float s0 = a + ab[(f * J + j) * H2 + 2 * h + 1];
      lin[(h * J + i) * J + j] = s0;
      float s = (s0 >= 0.f) ? s0 : 0.2f * s0;
      row[j] = s; mx = fmaxf(mx, s);
    }
    float sum = 0.f;
    for (int j = 0; j < J; ++j) { float e = expf(row[j] - mx); row[j] = e; sum += e; }
    float inv = 1.f / sum;
    for (int j = 0; j < J; ++j) {
      row[j] *= inv;
      att[(h * J + i) * J + j] = row[j] + ck[(h * J + i) * J + j];
    }
  }
  __syncthreads();
  // datt[h][i][j] = sum_{c in head} dY[i,c] G[j,c]
  for (int t = threadIdx.x; t < H * JJ; t += blockDim.x) {
    int h = t / JJ, r = t - h * JJ;
    int i = r / J, j = r - i * J;
    float s = 0.f;
    for (int c = 0; c < Cg; ++c)
      s = fmaf(dY[(f * J + i) * lddy + h * Cg + c], G[(f * J + j) * ldg + h * Cg + c], s);
    datt[t] = s;
    dCk_part[f * (long long)(H * JJ) + t] = s;
  }
  // dG[j,n] = sum_i att[h][i][j] dY[i,n]
  const int Ng = H * Cg;
  for (int t = threadIdx.x; t < J * Ng; t += blockDim.x) {
    int j = t / Ng, n = t - j * Ng;
    int h = n / Cg;
    float s = 0.f;
    for (int i = 0; i < J; ++i) s = fmaf(att[(h * J + i) * J + j], dY[(f * J + i) * lddy + n], s);
    dG[(f * J + j) * lddg + n] = s;
  }
  __syncthreads();
  // softmax + LeakyReLU backward -> dlin (in place in datt)
  for (int t = threadIdx.x; t < H * J; t += blockDim.x) {
    int h = t / J, i = t - h * J;
    float dot = 0.f;
    for (int j = 0; j < J; ++j) dot += P[(h * J + i) * J + j] * datt[(h * J + i) * J + j];
    for (int j = 0; j < J; ++j) {
      float ds = P[(h * J + i) * J + j] * (datt[(h * J + i) * J + j] - dot);
      float s0 = lin[(h * J + i) * J + j];
      datt[(h * J + i) * J + j] = (s0 >= 0.f) ? ds : 0.2f * ds;
    }
  }
  __syncthreads();
  // da_i = sum_j dlin[i][j] ; db_j = sum_i dlin[i][j]
  for (int t = threadIdx.x; t < H * J; t += blockDim.x) {
    int h = t / J, i = t - h * J;
    float da = 0.f, db = 0.f;
    for (int j = 0; j < J; ++j) {
      da += datt[(h * J + i) * J + j];
      db += datt[(h * J + j) * J + i];
    }
    dab[(f * J + i) * H2 + 2 * h] = da;
    dab[(f * J + i) * H2 + 2 * h + 1] = db;
  }
}

// dX[m][k] += sum_q dab[m][q] U[q][k]        (adjoint of the collapsed theta/phi row dots)
__global__ void rowdot_bwd_x_kernel(const float* __restrict__ dab, const float* __restrict__ U, int Q, long long M,
                                    int K, float* __restrict__ dX, int ldx) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * K) return;
  long long m = idx / K;
  int k = (int)(idx - m * K);
  float s = 0.f;
  for (int q = 0; q < Q; ++q) s = fmaf(dab[m * Q + q], U[(long long)q * K + k], s);
  dX[m * ldx + k] += s;
}

// parameter gradients of one head from dU (2 rows) and dcab (2 values); see global_collapse_kernel
__global__ void global_collapse_bwd_kernel(const float* __restrict__ dU, const float* __restrict__ dcab, int h, int C,
                                           int Ci, const float* __restrict__ tw, const float* __restrict__ tb,
                                           const float* __restrict__ pw, const float* __restrict__ pb,
                                           const float* __restrict__ wc, float* __restrict__ g_tw,
                                           float* __restrict__ g_tb, float* __restrict__ g_pw, float* __restrict__ g_pb,
                                           float* __restrict__ g_wc) {
  // one block per inter-channel m, the C input channels over the threads (coalesced rows, block reduction)
  const int m = blockIdx.x;
  if (m >= Ci) return;
  const float* du_t = dU + (long long)(2 * h) * C;
  const float* du_p = dU + (long long)(2 * h + 1) * C;
  const float wt = wc[m], wp = wc[Ci + m];
  float dwt = 0.f, dwp = 0.f;
  for (int k = threadIdx.x; k < C; k += blockDim.x) {
    const float ut = du_t[k], up = du_p[k];
    g_tw[(long long)m * C + k] = wt * ut;
    g_pw[(long long)m * C + k] = wp * up;
    dwt = fmaf(tw[(long long)m * C + k], ut, dwt);
    dwp = fmaf(pw[(long long)m * C + k], up, dwp);
  }
  __shared__ float red[2][32];
  dwt = warp_sum(dwt); dwp = warp_sum(dwp);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) { red[0][w] = dwt; red[1][w] = dwp; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = tb[m] * dcab[2 * h], b = pb[m] * dcab[2 * h + 1];
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) { a += red[0][i]; b += red[1][i]; }
    g_tb[m] = wt * dcab[2 * h];
    g_pb[m] = wp * dcab[2 * h + 1];
    g_wc[m] = a;
    g_wc[Ci + m] = b;
  }
}

// shrink adjoints (N = 3): dX[m][k] = sum_o dy[m][o] Ws[o][k] ; dWs[o][k] = sum_m dy[m][o] X[m][k]
__global__ void shrink_bwd_x_kernel(const float* __restrict__ dy, const float* __restrict__ Ws, long long M, int K,
                                    float* __restrict__ dX) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * K) return;
  long long m = idx / K;
  int k = (int)(idx - m * K);
  dX[idx] = dy[m * 3] * Ws[k] + dy[m * 3 + 1] * Ws[K + k] + dy[m * 3 + 2] * Ws[2 * K + k];
}
// block = 32 columns k x SBW_RG row groups; fixed-order reduction over the row groups (deterministic).  (One thread per
// output walking all M rows serially took 0.32 ms per step at b = 128: 3.5 % of the step for a 3 x 1024 matrix.)
constexpr int SBW_RG = 16;
__global__ void __launch_bounds__(32 * SBW_RG)
shrink_bwd_w_kernel(const float* __restrict__ dy, const float* __restrict__ X, long long M, int K,
                    float* __restrict__ dWs) {
  __shared__ double part[SBW_RG][3][33];
  const int kx = threadIdx.x, rg = threadIdx.y;
  const int k = blockIdx.x * 32 + kx;
  double s0 = 0.0, s1 = 0.0, s2 = 0.0;
  if (k < K) {
#pragma unroll 4
    for (long long m = rg; m < M; m += SBW_RG) {
      const double x = (double)X[m * K + k];
      s0 += (double)__ldg(dy + m * 3 + 0) * x;
      s1 += (double)__ldg(dy + m * 3 + 1) * x;
      s2 += (double)__ldg(dy + m * 3 + 2) * x;
    }
  }
  part[rg][0][kx] = s0; part[rg][1][kx] = s1; part[rg][2][kx] = s2;
  __syncthreads();
  if (rg < 3 && k < K) {
    double t = 0.0;
#pragma unroll
    for (int i = 0; i < SBW_RG; ++i) t += part[i][rg][kx];
    dWs[(long long)rg * K + k] = (float)t;
  }
}

// conv weight gradient re-layout: GEMM order [n][tap*Cin + c]  ->  parameter order (n, c, tap)
__global__ void conv_wgrad_relayout_kernel(const float* __restrict__ g, int N, int Cin, int taps, int ldg,
                                           float* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)N * Cin * taps) return;
  int n = (int)(idx / ((long long)Cin * taps));
  int rem = (int)(idx - (long long)n * Cin * taps);
  int c = rem / taps, tp = rem - c * taps;
  out[idx] = g[(long long)n * ldg + tp * Cin + c];
}

// SemCH weight gradient re-layout: stacked [(w, cout)][cin]  ->  parameter W (2, Cin, Cout)
__global__ void semch_wgrad_relayout_kernel(const float* __restrict__ g, int Cin, int Cout, int ldg,
                                            float* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)2 * Cin * Cout) return;
  int w = (int)(idx / ((long long)Cin * Cout));
  int rem = (int)(idx - (long long)w * Cin * Cout);
  int k = rem / Cout, c = rem - k * Cout;
  out[idx] = g[(long long)(w * Cout + c) * ldg + k];
}

// stacked SemCH weights for training: Wst[(w, cout)][cin] = W[w][cin][cout]
__global__ void semch_wstack_kernel(const float* __restrict__ W, int Cin, int Cout, float* __restrict__ out) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)2 * Cin * Cout) return;
  int r = (int)(idx / Cin), k = (int)(idx - (long long)r * Cin);
  int w = r / Cout, c = r - w * Cout;
  out[idx] = W[((long long)w * Cin + k) * Cout + c];
}

}  // namespace gast
