// Tensor-core GEMM core of the lifting path (sm_90a): TF32 on wgmma, in two precisions (template PREC).
//
//   TC_3XTF32 (default, fp32-grade):  D[128 rows, 128 cols] = A_hi.B_hi + A_lo.B_hi + A_hi.B_lo
//   TC_1XTF32 (opt-in, gast_set_precision(h, 1)):  D = A_hi.B_hi
//
// where x_hi = tf32(x) and x_lo = tf32(x - x_hi).  The dropped A_lo.B_lo term is 2^-22 of the result, so the
// 3xTF32 D matches an fp32 FFMA GEMM to ~1e-7 relative (the parity bar is 1e-4 abs; a single TF32 pass does
// not reach it, SURVEY.md §7).  The single pass is a third of the tensor work per multiply-add; its operands are
// rounded to 10 mantissa bits, and it is offered for inference only (DESIGN.md §4.1).
//
// The two forms share everything below except the slot contents (B_lo is not staged in 1xTF32), the ring depth
// and the number of wgmmas per k8 step (3 or 1).
//
// Two-level accumulation: the tensor core aligns and truncates its addends, so a long chain of MMAs
// into one accumulator is biased towards zero by ~0.5 ulp per MMA.  Every 16 K are therefore accumulated in a
// fresh register tile (6 wgmmas in 3xTF32, 2 in 1xTF32) and added into the fp32 tile sum with round-to-nearest (32 K per partial sum
// roughly doubled the error and pushed single training gradients past their bar).
//
// Per CTA (384 threads = 3 warpgroups, one CTA per SM), warp-specialised around a shared-memory ring of
// 32-wide K stages (3xTF32: 3 slots of B_hi | B_lo | A; 1xTF32: tc_stages(TC_1XTF32) slots of B_hi | A):
//   producer (warpgroup 0, 40 registers after setmaxnreg): waits for a slot's `empty` mbarrier, then fills it.
//     B (weights): the hi and lo copies are stored [K/4][N][4] (tc_prepare_weights), so one 3D TMA box per operand
//                lands in the no-swizzle K-major core-matrix layout wgmma reads from shared memory (8 rows x 16 B
//                core matrices, 128 B apart along N, 2048 B apart along K); one elected thread issues the boxes.
//     A (activations): rows are gathered per frame (dilated / strided taps, residual slices, concatenations), so
//                they arrive by cp.async (16 B per row and k-quad, zero-filled outside the tile) from all 128
//                producer threads.  A stage never straddles a tap (Kc % 32 == 0), so segment, tap and column are
//                advanced once per stage.
//     The slot's `full` mbarrier completes when the TMA bytes (expect_tx) and every producer thread's cp.asyncs
//     (cp.async.mbarrier.arrive.noinc) have landed: 1 + 128 arrivals.
//   consumers (warpgroups 1 and 2, 232 registers): warpgroup 1 + w owns rows 64w .. 64w+63 and all 128 columns:
//     wgmma.m64n128k8 tf32, A from registers (loaded from the slot and converted to tf32 there, split into hi / lo in
//     3xTF32), B from the shared-memory descriptor.  A stage's two 16-K partials go into two register tiles back to back;
//     the first is added into the tile sum while the second runs (wgmma.wait_group 1), then the second is retired
//     and added, and the slot is released (its `empty` mbarrier, one arrival per consumer warp, 8 in all).  No
//     partial stays in flight across the loop's back edge: ptxas then serialises every wgmma of the kernel (C7514).
//     The two consumers do not synchronise with each other inside the K loop, so one's MMAs fill the other's drain.
// Tiles (fpt whole frames per 128-row tile) and the fused epilogues (gemm_epilogue, run by the 256 consumer threads)
// are the FFMA core's, so both cores are interchangeable per launch.
//
// One tile per CTA, on a 1D grid in which the column tile is the fast index (tc_launch): the CTAs dispatched together
// cover a row tile's column tiles side by side, so its A rows come from HBM once and its other column tiles find them
// in L2.  (Every layer's A is larger than the L2; with the row tile fast, A was read from HBM once per column tile.)
#pragma once
#include <cuda.h>
#include <vector>
#include "gast_common.cuh"
#include "gemm_ffma.cuh"

namespace gast {

struct TcWeights {
  float* hi = nullptr;   // tf32(W), stored [K/4][N][4]
  float* lo = nullptr;   // tf32(W - tf32(W)), same layout
  CUtensorMap map_hi, map_lo;
  int N = 0, K = 0;
  bool ready = false;
};

enum { TC_3XTF32 = 0, TC_1XTF32 = 1 };               // precision of the core: gast_set_precision's mode

#ifndef GAST_TC1_STAGES
#define GAST_TC1_STAGES 3                             // ring depth of the 1xTF32 form: 4 and 5 measured slower (DESIGN.md §4.1)
#endif

constexpr int TC_BM = 128, TC_BN = 128;
constexpr int TC_KS = 32;                            // K per ring stage; segment widths must be multiples of it
constexpr int TC_KP = 16;                            // K per partial sum, added into the tile sum with RN
constexpr int TC_THREADS = 384;                      // warpgroup 0 produces, warpgroups 1 and 2 consume
constexpr int TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;   // 128 * 40 + 256 * 232 <= 64K registers of the SM
constexpr int TC_ALD = TC_KS + 4;                    // A stage row stride (floats): conflict-free fragment loads
constexpr int TC_B_BYTES = TC_BN * TC_KS * 4;        // one of B_hi / B_lo in a stage
constexpr int TC_A_BYTES = TC_BM * TC_ALD * 4;
// B copies per slot, slot size and ring depth of each precision.  3xTF32: a fourth slot measured slower
// (DESIGN.md §4.1).
__host__ __device__ constexpr int tc_nb(int prec) { return prec == TC_1XTF32 ? 1 : 2; }
__host__ __device__ constexpr int tc_slot(int prec) { return tc_nb(prec) * TC_B_BYTES + TC_A_BYTES; }   // B_hi [| B_lo] | A
__host__ __device__ constexpr int tc_stages(int prec) { return prec == TC_1XTF32 ? GAST_TC1_STAGES : 3; }
__host__ __device__ constexpr int tc_ring(int prec) { return tc_stages(prec) * tc_slot(prec); }
constexpr int TC_STG_LD = 136;                       // [row][col] stride of the accumulator hand-over to the epilogue
constexpr int TC_ROWBASE_BYTES = 3 * 128 * sizeof(long long);
constexpr int TC_SMEM_MAX = 200 * 1024;
static_assert(tc_slot(TC_3XTF32) % 1024 == 0 && tc_slot(TC_1XTF32) % 1024 == 0, "ring slots stay 1024-byte aligned");
static_assert(tc_ring(TC_1XTF32) + 16 * tc_stages(TC_1XTF32) + TC_ROWBASE_BYTES + 1024 <= TC_SMEM_MAX,
              "the 1xTF32 ring fits the shared memory the 3xTF32 form may use");

__host__ __device__ inline size_t tc_smem_bytes(int prec, int epi, int J, int fpt, int hpt) {
  size_t m = (size_t)tc_ring(prec) + 16 * tc_stages(prec);   // + a full and an empty mbarrier per slot
  const size_t stg = (size_t)TC_BM * TC_STG_LD * 4;
  const size_t e = ffma_smem_bytes(epi, J, fpt, hpt) - TC_ROWBASE_BYTES;
  if (stg > m) m = stg;
  if (e > m) m = e;
  return TC_ROWBASE_BYTES + 1024 + m;                // + alignment of the ring to 1024 bytes
}

__device__ __forceinline__ uint32_t tf32_bits(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y), "r"(z) : "memory");
}
// 16 bytes global -> shared, zero-filled when src_bytes == 0
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// arrive on `bar` once every cp.async this thread has issued so far has landed (counted in the barrier's init count)
__device__ __forceinline__ void cp_async_arrive(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// shared-memory matrix descriptor of a no-swizzle K-major operand: core matrices 128 B apart along N (SBO),
// 2048 B apart along K (LBO)
__device__ __forceinline__ uint64_t tc_bdesc(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)(2048 >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins a register tile at this point of the program, so that the compiler does not move its reads or writes across
// the wgmma fence / commit / wait around it
__device__ __forceinline__ void tile_fence(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

// d (+)= a . B, m64n128k8, tf32 operands (A from registers, B from shared memory), fp32 accumulate;
// scale_d == 0 overwrites d
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %68, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %69, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(scale_d), "l"(bdesc));
}

// One 16-K partial of a consumer: d = sum over the k8 steps s0, s0 + 1 of the slot at sb of
// A_lo.B_hi + A_hi.B_lo + A_hi.B_hi (3xTF32, small products first) or A_hi.B_hi (1xTF32), issued as one wgmma group
template <int PREC>
__device__ __forceinline__ void tc_partial(float (&d)[64], const uint32_t (&ah)[2][4], const uint32_t (&al)[2][4],
                                           uint32_t sb, int s0) {
  tile_fence(d);
  wgmma_fence();
#pragma unroll
  for (int i = 0; i < 2; ++i) {   // k8 step s = core matrices 2s, 2s+1
    const int s = s0 + i;
    const uint64_t dh = tc_bdesc(sb + s * 4096);
    if (PREC == TC_3XTF32) {
      const uint64_t dl = tc_bdesc(sb + TC_B_BYTES + s * 4096);
      wgmma_tf32(d, al[i], dh, i);
      wgmma_tf32(d, ah[i], dl, 1);
      wgmma_tf32(d, ah[i], dh, 1);
    } else {
      wgmma_tf32(d, ah[i], dh, i);
    }
  }
  wgmma_commit();
}

// A fragment rows r0, r0 + 8 of the k8 steps s0, s0 + 1 of a slot's A (row stride TC_ALD), rounded to tf32 (hi) and,
// in 3xTF32, the rounding error split off as lo
template <int PREC>
__device__ __forceinline__ void tc_load_a(const float* A, int r0, int t, int s0, uint32_t (&ah)[2][4],
                                          uint32_t (&al)[2][4]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int k = 8 * (s0 + i) + t;
    const float x[4] = {A[r0 * TC_ALD + k], A[(r0 + 8) * TC_ALD + k], A[r0 * TC_ALD + k + 4],
                        A[(r0 + 8) * TC_ALD + k + 4]};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      ah[i][q] = tf32_bits(x[q]);
      if (PREC == TC_3XTF32) al[i][q] = tf32_bits(x[q] - __uint_as_float(ah[i][q]));
    }
  }
}

__device__ __forceinline__ void tc_add(float (&acc)[64], float (&part)[64]) {
  tile_fence(part);
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] += part[i];
}

// This CTA's row tile and column tile.  %ctaid is read with a volatile move, so that the consumers can recompute the
// tile after their K loop instead of keeping it in registers through it (that spilled in the SemCH instantiation).
__device__ __forceinline__ void tc_tile(const GemmP& p, int& rt, int& ctile) {
  uint32_t b;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(b));
  const int col_tiles = (p.N + TC_BN - 1) / TC_BN;
  rt = (int)b / col_tiles;
  ctile = (int)b - rt * col_tiles;
}

// mlo is not read in 1xTF32
template <int EPI, int PREC>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ GemmP p, const __grid_constant__ CUtensorMap mhi,
               const __grid_constant__ CUtensorMap mlo) {
  constexpr int STAGES = tc_stages(PREC), SLOT = tc_slot(PREC), NB = tc_nb(PREC);
  extern __shared__ __align__(16) unsigned char smem_raw[];
  long long* rowbase = reinterpret_cast<long long*>(smem_raw);          // [3][128]
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t rb = (raw + TC_ROWBASE_BYTES + 1023) & ~1023u;        // ring base (shared address)
  unsigned char* ring = smem_raw + (rb - raw);
  const uint32_t full0 = rb + tc_ring(PREC);                            // per ring slot: stage landed
  const uint32_t empty0 = full0 + 8 * STAGES;                           // per ring slot: both consumers done with it

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int J = p.J;
  int rt, ctile;
  tc_tile(p, rt, ctile);
  const int f0 = rt * p.fpt;
  const int nf = min(p.fpt, p.F - f0);
  const int vrows = nf * J;
  const int n0 = ctile * TC_BN;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, 1 + 128);
      mbar_init(empty0 + 8 * s, 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  for (int i = tid; i < p.nseg * 128; i += TC_THREADS) {
    int s = i >> 7, r = i & 127;
    long long off = -1;
    if (r < vrows) {
      int fr = r / J, j = r - fr * J;
      long long fin = map_frame(p.seg[s].map, f0 + fr);
      off = (fin * J + j) * (long long)p.seg[s].ld;
    }
    rowbase[s * 128 + r] = off;
  }
  __syncthreads();

  int nstages = 0;
  for (int s = 0; s < p.nseg; ++s) nstages += p.seg[s].K / TC_KS;

  if (warp < 4) {
    // producer: stage c into ring slot c % STAGES once both consumers have released the slot's previous stage
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    const int q = tid & 7, rq = tid >> 3;                               // k-quad q of rows rq + 16 i
    int seg = 0, k0 = 0, kcol = 0, tap = 0, kin = 0;                    // stage start: segment, K in it, W column, tap
    for (int c = 0; c < nstages; ++c) {
      const int slot = c % STAGES;
      if (c >= STAGES) mbar_wait(empty0 + 8 * slot, (c / STAGES - 1) & 1);
      const uint32_t sb = rb + slot * SLOT, full = full0 + 8 * slot;
      if (tid == 0) {
        mbar_arrive_expect_tx(full, NB * TC_B_BYTES);
        const int kq = (kcol + k0) >> 2;
        tma_load_3d(sb, &mhi, full, 0, n0, kq);
        if (NB == 2) tma_load_3d(sb + TC_B_BYTES, &mlo, full, 0, n0, kq);
      }
      const ASeg& sg = p.seg[seg];
      const float* src = sg.base + tap * sg.tap_stride + kin + q * 4;
#pragma unroll
      for (int i = 0; i < TC_BM / 16; ++i) {
        const int r = rq + 16 * i;
        const long long off = rowbase[seg * 128 + r];
        cp_async16(sb + NB * TC_B_BYTES + (r * TC_ALD + q * 4) * 4, off >= 0 ? src + off : sg.base, off >= 0 ? 16 : 0);
      }
      cp_async_arrive(full);
      k0 += TC_KS;
      kin += TC_KS;
      if (kin == sg.Kc) { kin = 0; ++tap; }
      if (k0 == sg.K) { kcol += sg.K; k0 = 0; tap = 0; ++seg; }
    }
    cp_async_wait_all();
    return;
  }

  // consumers
  setmaxnreg_inc<TC_CONSUMER_REGS>();
  const int ct = tid - 128;                                             // 0 .. 255: the epilogue's thread index
  const int wg = ct >> 7, wq = (ct >> 5) & 3;
  const int g = lane >> 2, t = lane & 3;
  const int r0 = wg * 64 + wq * 16 + g;                                 // fragment rows r0 and r0 + 8
  float acc[64], part0[64], part1[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;

  for (int c = 0; c < nstages; ++c) {
    const int slot = c % STAGES;
    mbar_wait(full0 + 8 * slot, (c / STAGES) & 1);
    const uint32_t sb = rb + slot * SLOT;
    const float* A = reinterpret_cast<const float*>(ring + slot * SLOT + NB * TC_B_BYTES);
    uint32_t ah[2][4], al[2][4];
    tc_load_a<PREC>(A, r0, t, 0, ah, al);
    tc_partial<PREC>(part0, ah, al, sb, 0);
    tc_load_a<PREC>(A, r0, t, 2, ah, al);
    tc_partial<PREC>(part1, ah, al, sb, 2);
    wgmma_wait<1>();                            // the first partial has retired ...
    tc_add(acc, part0);                         // ... and is summed while the second runs
    wgmma_wait<0>();
    tc_add(acc, part1);
    if (lane == 0) mbar_arrive(empty0 + 8 * slot);
  }
  epi_sync();                                   // both consumers are done with the ring
  tc_tile(p, rt, ctile);
  const int fe = rt * p.fpt, nfe = min(p.fpt, p.F - fe);

  // hand the tile over in the FFMA thread layout the shared epilogues expect
  float* S = reinterpret_cast<float*>(ring);   // [128][TC_STG_LD]
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int col = 8 * i + 2 * t;
    *reinterpret_cast<float2*>(S + r0 * TC_STG_LD + col) = make_float2(acc[4 * i], acc[4 * i + 1]);
    *reinterpret_cast<float2*>(S + (r0 + 8) * TC_STG_LD + col) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
  }
  epi_sync();
  const int ty = ct >> 4, tx = ct & 15;
  float out[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4);
    const float4 u = *reinterpret_cast<const float4*>(S + r * TC_STG_LD + tx * 4);
    const float4 v = *reinterpret_cast<const float4*>(S + r * TC_STG_LD + 64 + tx * 4);
    out[i][0] = u.x; out[i][1] = u.y; out[i][2] = u.z; out[i][3] = u.w;
    out[i][4] = v.x; out[i][5] = v.y; out[i][6] = v.z; out[i][7] = v.w;
  }
  epi_sync();
  gemm_epilogue<EPI>(p, out, reinterpret_cast<float*>(ring), ct, fe, nfe, nfe * J, ctile * TC_BN, ctile);
}

// W [N][K] -> hi / lo in the TMA-friendly layout [K/4][N][4] (both precisions read hi = tf32(W))
__global__ void tc_split_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int N, int K) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * K) return;
  const int n = (int)(i / K), k = (int)(i - (long long)n * K);
  const float x = w[i];
  const float h = __uint_as_float(tf32_bits(x));
  const long long o = ((long long)(k >> 2) * N + n) * 4 + (k & 3);
  hi[o] = h;
  lo[o] = __uint_as_float(tf32_bits(x - h));
}

typedef CUresult (*tc_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                 const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                 CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline tc_encode_fn tc_get_encode() {
  static tc_encode_fn fn = nullptr;
  if (!fn) {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<tc_encode_fn>(q);
  }
  return fn;
}

// W: [N][K] fp32 K-major (device).  Allocates hi / lo once per shape, encodes their TMA maps and splits W into them.
// Returns 0 on success (t.ready says whether the core takes the shape), a cudaError_t or -1 otherwise.
inline int tc_prepare_weights(TcWeights& t, const float* W, int N, int K, cudaStream_t st, std::vector<void*>* owned) {
  t.ready = false;
  if (K % TC_KS != 0 || N % 4 != 0) return 0;            // shape not taken by this core (FFMA runs it)
  if (!t.hi || t.N != N || t.K != K) {
    tc_encode_fn enc = tc_get_encode();
    if (!enc) return -1;
    void* a = nullptr; void* b = nullptr;
    cudaError_t e = cudaMalloc(&a, sizeof(float) * (size_t)N * K);
    if (e != cudaSuccess) return (int)e;
    e = cudaMalloc(&b, sizeof(float) * (size_t)N * K);
    if (e != cudaSuccess) { cudaFree(a); return (int)e; }
    owned->push_back(a); owned->push_back(b);
    t.hi = (float*)a; t.lo = (float*)b; t.N = N; t.K = K;
    // dims {4 k's, N rows, K/4 k-quads}; box {4, 128, TC_KS/4}: rows past N read as zero
    cuuint64_t dims[3] = {4, (cuuint64_t)N, (cuuint64_t)(K / 4)};
    cuuint64_t strides[2] = {16, (cuuint64_t)N * 16};
    cuuint32_t box[3] = {4, (cuuint32_t)TC_BN, (cuuint32_t)(TC_KS / 4)};
    cuuint32_t estr[3] = {1, 1, 1};
    for (int m = 0; m < 2; ++m) {
      CUresult r = enc(m ? &t.map_lo : &t.map_hi, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, m ? t.lo : t.hi, dims, strides, box,
                       estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { t.hi = nullptr; return -1; }
    }
  }
  const long long n = (long long)N * K;
  tc_split_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, t.hi, t.lo, N, K);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  t.ready = true;
  return 0;
}

// The shapes the core takes are the same in both precisions (the 1xTF32 ring is no larger than the bound below).
inline bool tc_supported(const GemmP& p, int epi, const TcWeights& t) {
  if (!t.ready || t.K != p.ldw || t.N < p.N || p.N % 4) return false;
  for (int s = 0; s < p.nseg; ++s) {
    const ASeg& sg = p.seg[s];
    if (sg.K % TC_KS || sg.Kc % TC_KS || sg.ld % 4 || sg.tap_stride % 4) return false;
    if (reinterpret_cast<uintptr_t>(sg.base) & 15) return false;
  }
  const int hpt = epi == EPI_GLOBAL ? (p.heads < 4 ? p.heads : 4) : 1;
  if (tc_smem_bytes(TC_3XTF32, epi, p.J, p.fpt, hpt) > TC_SMEM_MAX) return false;
  if (tc_smem_bytes(TC_1XTF32, epi, p.J, p.fpt, hpt) > TC_SMEM_MAX) return false;
  return true;
}

template <int PREC>
inline int tc_launch_prec(cudaStream_t st, int epi, const GemmP& p, const TcWeights& t) {
  const dim3 grid((unsigned)(((p.F + p.fpt - 1) / p.fpt) * ((p.N + TC_BN - 1) / TC_BN)));
  const int hpt = epi == EPI_GLOBAL ? (p.heads < 4 ? p.heads : 4) : 1;
  const size_t smem = tc_smem_bytes(PREC, epi, p.J, p.fpt, hpt);
  static bool attr_set[64][3];              // the shared-memory opt-in is per device
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63][epi]) {
    const void* fn = epi == EPI_PLAIN ? (const void*)gemm_tc_kernel<EPI_PLAIN, PREC>
                   : epi == EPI_SEMCH ? (const void*)gemm_tc_kernel<EPI_SEMCH, PREC>
                                      : (const void*)gemm_tc_kernel<EPI_GLOBAL, PREC>;
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev & 63][epi] = true;
  }
  if (epi == EPI_PLAIN) gemm_tc_kernel<EPI_PLAIN, PREC><<<grid, TC_THREADS, smem, st>>>(p, t.map_hi, t.map_lo);
  else if (epi == EPI_SEMCH) gemm_tc_kernel<EPI_SEMCH, PREC><<<grid, TC_THREADS, smem, st>>>(p, t.map_hi, t.map_lo);
  else gemm_tc_kernel<EPI_GLOBAL, PREC><<<grid, TC_THREADS, smem, st>>>(p, t.map_hi, t.map_lo);
  return (int)cudaGetLastError();
}

// One CTA per tile, tile = row tile * column tiles + column tile (the column tile fastest, see gemm_tc_kernel).
// prec: TC_3XTF32 or TC_1XTF32.
inline int tc_launch(cudaStream_t st, int epi, const GemmP& p, const TcWeights& t, int prec) {
  return prec == TC_1XTF32 ? tc_launch_prec<TC_1XTF32>(st, epi, p, t) : tc_launch_prec<TC_3XTF32>(st, epi, p, t);
}

}  // namespace gast
