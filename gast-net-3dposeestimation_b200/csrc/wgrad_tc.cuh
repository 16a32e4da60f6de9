// TF32 weight gradient on wgmma (sm_90a): dW[N][K] = sum over the rows m of dZ[m][N]^T . A[m][K], the contraction of
// dense_tn (train.cuh) in the opt-in training precision (gast_set_train_precision(h, 1)).
//
// Same tiles and splits as wgrad_tn_kernel: a CTA owns a 128 x 128 tile of dW and one row range of the split; its
// partial goes to part + split * N * K and wgrad_reduce_kernel sums the partials in split order, so the result repeats
// bit for bit.  The wgmma roles: M = 128 dW rows (n, two warpgroups of 64), N = 128 dW columns (k), K = the rows m.
//   A operand (dZ^T, registers): the 64 x 8 fragment of a k8 step is dZ[m][n] with m along the fragment's K, so the
//     dZ slab is staged row-major as it lies in memory ([32 rows][128 + 8 floats]: the fragment loads of a warp hit
//     32 different banks) and read into registers, rounded with cvt.rna.tf32.f32.
//   B operand (A, shared memory): wgmma takes tf32 only K-major, i.e. 4 consecutive m of one column k in 16 bytes.
//     The A slab is transposed on its way in: every element is its own 4-byte cp.async into [m/4][k][m%4] (the
//     layout gemm_tc_kernel's weights have, read by the same descriptor, tc_bdesc).  A warp's 32 copies are 4 rows
//     x 8 columns, so its global reads fill 32-byte sectors and its shared-memory writes are one contiguous 128 bytes.
//     The B operand is rounded by the tensor core itself, which reads only the tf32 bits (truncation); to round to
//     nearest as the forward's TC_1XTF32 does, the staged slab is rounded in place (cvt.rna) before the MMAs read it.
//   Rows past the split's end and columns past N / K are zero-filled (cp.async with 0 source bytes).
// Accumulation is the forward core's two-level scheme: each 16 rows of m go into a fresh register tile (two k8 wgmmas)
// that is added into the fp32 tile sum with round-to-nearest; a 32-row stage issues both 16-row partials back to back.
// Three ring stages of cp.async groups, one __syncthreads per stage.
// Shapes: N % 32 == 0 and K % 32 == 0 (so the 8-wide dab contraction and the expand conv's KP stay on
// wgrad_tn_kernel), dZ 16-byte aligned with lddz % 4 == 0; any M and any split.
#pragma once
#include "gemm_tc.cuh"
#include "train_kernels.cuh"

namespace gast {

constexpr int WT_MS = 32;                                // rows of m per stage: two 16-row partials
constexpr int WT_STAGES = 3;
constexpr int WT_THREADS = 256;                          // two consumer warpgroups, both also copy
constexpr int WT_ZLD = WG_T + 8;                         // dZ slab row stride (floats)
constexpr int WT_B_BYTES = WT_MS * WG_T * 4;             // transposed A slab [m/4][k][4]
constexpr int WT_Z_BYTES = WT_MS * WT_ZLD * 4;
constexpr int WT_STAGE_BYTES = WT_B_BYTES + WT_Z_BYTES;
constexpr int WT_SMEM = WT_STAGES * WT_STAGE_BYTES + 128;
static_assert(WT_B_BYTES % 128 == 0 && WT_STAGE_BYTES % 128 == 0, "descriptor bases stay 128-byte aligned");

// 4 bytes global -> shared, zero-filled when src_bytes == 0
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}

// A fragment (dZ^T) rows r0, r0 + 8 of the k8 steps s0, s0 + 1 of a dZ slab, rounded to tf32
__device__ __forceinline__ void wt_load_a(const float* Z, int r0, int t, int s0, uint32_t (&a)[2][4]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = 8 * (s0 + i) + t;
    a[i][0] = tf32_bits(Z[m * WT_ZLD + r0]);
    a[i][1] = tf32_bits(Z[m * WT_ZLD + r0 + 8]);
    a[i][2] = tf32_bits(Z[(m + 4) * WT_ZLD + r0]);
    a[i][3] = tf32_bits(Z[(m + 4) * WT_ZLD + r0 + 8]);
  }
}

__global__ void __launch_bounds__(WT_THREADS, 1)
wgrad_tc_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ A, int lda, long long M, int N,
                int K, long long rows_per_split, float* __restrict__ part) {
  extern __shared__ __align__(16) unsigned char wt_smem[];
  const uint32_t raw = smem_u32(wt_smem);
  const uint32_t base = (raw + 127) & ~127u;
  unsigned char* sm = wt_smem + (base - raw);
  const int n0 = blockIdx.x * WG_T, k0 = blockIdx.y * WG_T;
  const long long m_beg = (long long)blockIdx.z * rows_per_split;
  const long long m_end = min(M, m_beg + rows_per_split);
  const int nst = m_end > m_beg ? (int)((m_end - m_beg + WT_MS - 1) / WT_MS) : 0;
  const int tid = threadIdx.x, lane = tid & 31;

  // copies of stage c into ring slot c % WT_STAGES.  dZ: 16-byte chunks tid + 256 i of the 32 x 128 slab.  A: element
  // 256 i + tid of the transposed slab, i.e. row 4 (i / 2) + tid % 4, column 64 (i % 2) + tid / 4.
  auto issue = [&](int c) {
    const uint32_t sb = base + (c % WT_STAGES) * WT_STAGE_BYTES;
    const long long m0 = m_beg + (long long)c * WT_MS;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int ch = tid + 256 * i, r = ch >> 5, q = (ch & 31) * 4;
      const bool ok = m0 + r < m_end && n0 + q < N;
      cp_async16(sb + WT_B_BYTES + (r * WT_ZLD + q) * 4, ok ? dZ + (m0 + r) * lddz + n0 + q : dZ, ok ? 16 : 0);
    }
    const int ar = tid & 3, aj = tid >> 2;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int r = 4 * (i >> 1) + ar, j = 64 * (i & 1) + aj;
      const bool ok = m0 + r < m_end && k0 + j < K;
      cp_async4(sb + (((r >> 2) * WG_T + j) * 4 + ar) * 4, ok ? A + (m0 + r) * lda + k0 + j : A, ok ? 4 : 0);
    }
  };

  const int wg = tid >> 7, wq = (tid >> 5) & 3, g = lane >> 2, t = lane & 3;
  const int r0 = wg * 64 + wq * 16 + g;                 // fragment rows r0 and r0 + 8 = dW rows n0 + r0, n0 + r0 + 8
  float acc[64], part0[64], part1[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

#pragma unroll
  for (int c = 0; c < WT_STAGES - 1; ++c) {
    if (c < nst) issue(c);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int c = 0; c < nst; ++c) {
    asm volatile("cp.async.wait_group %0;" ::"n"(WT_STAGES - 2) : "memory");   // this thread's copies of stage c
    // round the B slab to nearest tf32 in place (each thread its own 16 elements of the stage)
    const int slot = c % WT_STAGES;
    float* Bs = reinterpret_cast<float*>(sm + slot * WT_STAGE_BYTES);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int r = 4 * (i >> 1) + (tid & 3), j = 64 * (i & 1) + (tid >> 2);
      float& v = Bs[((r >> 2) * WG_T + j) * 4 + (r & 3)];
      v = __uint_as_float(tf32_bits(v));
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> wgmma's reads
    __syncthreads();   // stage c landed for every thread, and every thread is done with stage c - 1's slot
    if (c + WT_STAGES - 1 < nst) issue(c + WT_STAGES - 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    const uint32_t sb = base + slot * WT_STAGE_BYTES;
    const float* Z = reinterpret_cast<const float*>(sm + slot * WT_STAGE_BYTES + WT_B_BYTES);
    uint32_t a[2][4], unused[2][4];
    wt_load_a(Z, r0, t, 0, a);
    tc_partial<TC_1XTF32>(part0, a, unused, sb, 0);
    wt_load_a(Z, r0, t, 2, a);
    tc_partial<TC_1XTF32>(part1, a, unused, sb, 2);
    wgmma_wait<1>();
    tc_add(acc, part0);
    wgmma_wait<0>();
    tc_add(acc, part1);
  }
  asm volatile("cp.async.wait_all;" ::: "memory");

  float* out = part + (long long)blockIdx.z * N * K;
  const int n = n0 + r0;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int k = k0 + 8 * i + 2 * t;
    if (k >= K) continue;
    if (n < N) *reinterpret_cast<float2*>(out + (long long)n * K + k) = make_float2(acc[4 * i], acc[4 * i + 1]);
    if (n + 8 < N)
      *reinterpret_cast<float2*>(out + (long long)(n + 8) * K + k) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
  }
}

// whether wgrad_tc_kernel takes the contraction (the shapes of the header comment)
inline bool wgrad_tc_takes(const float* dZ, int lddz, int N, int K) {
  return N % 32 == 0 && K % 32 == 0 && lddz % 4 == 0 && (reinterpret_cast<uintptr_t>(dZ) & 15) == 0;
}

// S splits of rps rows over the grid of wgrad_tn_kernel; returns a cudaError_t
inline int wgrad_tc_launch(cudaStream_t st, const float* dZ, int lddz, const float* A, int lda, long long M, int N,
                           int K, long long rps, long long S, float* part) {
  static bool attr_set[64];                  // the shared-memory opt-in is per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63]) {
    const cudaError_t e = cudaFuncSetAttribute((const void*)wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               WT_SMEM);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev & 63] = true;
  }
  const dim3 grid((unsigned)((N + WG_T - 1) / WG_T), (unsigned)((K + WG_T - 1) / WG_T), (unsigned)S);
  wgrad_tc_kernel<<<grid, WT_THREADS, WT_SMEM, st>>>(dZ, lddz, A, lda, M, N, K, rps, part);
  return (int)cudaGetLastError();
}

}  // namespace gast
