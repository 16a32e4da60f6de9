// Tensor-core GEMM core of the lifting path (sm_90a): wgmma in three precisions (template PREC).
//
//   TC_F16X3 (inference at fp32 grade, gast_set_precision(h, 0)):
//       D[128 rows, 128 cols] = 2^-(s_r + s_W) (A_lo.B_hi + A_hi.B_lo + A_hi.B_hi), fp16 operands
//   TC_3XTF32 (training and every gradient, fp32 grade):  D = A_hi.B_hi + A_lo.B_hi + A_hi.B_lo, tf32 operands
//   TC_1XTF32 (opt-in, gast_set_precision(h, 1)):  D = A_hi.B_hi, tf32 operands
//
// 3xTF32 / 1xTF32: x_hi = tf32(x) and x_lo = tf32(x - x_hi).  F16X3: x is first scaled by an exact power of two,
// 2^s_W per weight matrix (max |W| 2^s_W in [2^14, 2^15), tc_prepare_weights) and 2^s_r per A row and 32-K stage
// (chosen the same way from the row's 32 values, in the consumers), then x_hi = fp16(x 2^s) and
// x_lo = fp16(x 2^s - x_hi).  fp16 and tf32 both carry 11 significant bits, so both splits carry 22 and the dropped
// A_lo.B_lo term is 2^-22 of the result in either: D matches an fp32 FFMA GEMM to ~1e-7 relative (the parity bar is
// 1e-4 abs; a single TF32 pass does not reach it, SURVEY.md §7).  The scales keep fp32's range (no activation
// saturates at fp16's 65504) and add no rounding; 2^-(s_r + s_W) is applied when a 16-K partial is added into the
// tile sum, in the same single rounding as an add.  An fp16 product runs at twice the TF32 rate and stages half the
// weight bytes, so F16X3 costs half of 3xTF32 in tensor time and a third less in staged bytes.  The single TF32
// pass is a third of the 3xTF32 tensor work; its operands are rounded to 10 mantissa bits, and it is offered for
// inference only (DESIGN.md §4.1).
//
// The three forms share everything below except the slot contents (B_lo is not staged in 1xTF32; F16X3 stages
// fp16 B copies), the ring depth and the wgmmas per 16-K partial (3xTF32 6 m64n128k8, 1xTF32 2, F16X3 3 m64n128k16).
//
// Two-level accumulation: the tensor core aligns and truncates its addends, so a long chain of MMAs
// into one accumulator is biased towards zero by ~0.5 ulp per MMA.  Every 16 K are therefore accumulated in a
// fresh register tile and added into the fp32 tile sum with round-to-nearest (32 K per partial sum
// roughly doubled the error and pushed single training gradients past their bar).
//
// Per CTA (384 threads = 3 warpgroups, one CTA per SM), warp-specialised around a shared-memory ring of
// 32-wide K stages (tc_stages(PREC) slots of B_hi | B_lo | A, B_hi | A in 1xTF32):
//   producer (warpgroup 0, 40 registers after setmaxnreg): waits for a slot's `empty` mbarrier, then fills it.
//     B (weights): the hi and lo copies are stored [K/4][N][4] floats ([K/8][N][8] halves in F16X3,
//                tc_prepare_weights), so one TMA box per operand lands in the no-swizzle K-major core-matrix
//                layout wgmma reads from shared memory (8 rows x 16 B core matrices, 128 B apart along N, 2048 B
//                apart along K); the box is described as rows of 2 KB (a k-quad or k-octet of the tile's 128 n),
//                not 16-byte rows, and one elected thread issues the boxes.
//     A (activations): a stage is 128 dense rows of 32 floats in TMA's 128-byte swizzle (chunk c of row r at
//                c ^ (r & 7)), which keeps the consumers' fragment loads free of bank conflicts.  A segment whose
//                frame map is affine over the launch (tc_seg_tma: source frame t_mul f + t_off, tap k tap_stride
//                floats on; the 1x1 layers, SemCH, the attention GEMMs, the block concatenations, the strided stage
//                convolutions and a stream's ring taps) is one 4D TMA box {32, J, 1, fpt} per stage from the same
//                elected thread (tc_encode_taps): the tile's fpt J rows land densely from the slot's A, frames past F
//                zero-filled, slot rows past fpt J left as they were (they belong to no stored output row).  Rows
//                gathered per frame (the dilated schedule across clips, the streams' chunk calls) arrive by cp.async
//                (16 B per row and k-quad, zero-filled outside the tile) from all 128 producer threads into the same
//                swizzled layout.  A stage never straddles a tap (Kc % 32 == 0), so segment, tap, column and path are
//                chosen once per stage.
//     The slot's `full` mbarrier completes when the TMA bytes (expect_tx) and, in a launch with a gathered segment,
//     every producer thread's cp.asyncs (cp.async.mbarrier.arrive.noinc) or plain arrivals have landed: 1 + 128
//     arrivals; 1 when every segment is loaded by TMA (the other producer threads then leave at once).
//   consumers (warpgroups 1 and 2, 232 registers): warpgroup 1 + w owns rows 64w .. 64w+63 and all 128 columns:
//     wgmma.m64n128k8 tf32 or m64n128k16 f16, A from registers (loaded from the slot and converted there: to tf32,
//     split into hi / lo in 3xTF32; in F16X3 the four threads of a quad find their rows' max |a| over the stage's
//     32 K with two shuffles, scale and split into fp16 hi / lo), B from the shared-memory descriptor.  A stage's
//     two 16-K partials go into two register tiles back to back;
//     the first is added into the tile sum while the second runs (wgmma.wait_group 1), then the second is retired
//     and added, and the slot is released (its `empty` mbarrier, one arrival per consumer warp, 8 in all).  No
//     partial stays in flight across the loop's back edge: ptxas then serialises every wgmma of the kernel (C7514).
//     The two consumers do not synchronise with each other inside the K loop, so one's MMAs fill the other's drain.
// Tiles (fpt whole frames per 128-row tile) and the fused epilogues are the FFMA core's, so both cores are
// interchangeable per launch.  EPI_PLAIN and EPI_SEMCH run on the wgmma fragments, in gemm_epilogue's order, and leave
// by TMA tensor stores from a 64 KB staging buffer of their own: tc_store_plain (bias, ReLU, residual) stores four
// 32-column blocks.  An affine residual map (tc_res_tma: the stage 1x1 layers, a stream's residual slot) has the
// tile's residual loaded into that buffer by TMA during the K loop (tc_load_res: consumer thread 0 after the tile's
// third stage, on an mbarrier of its own), so the epilogue reads it from shared memory at the positions it then
// overwrites instead of from HBM after the K loop; tc_store_semch stages the neighbour half of the tile in two of the blocks, mixes each row's
// neighbours into the other two and stores those.  EPI_GLOBAL's attention mix is handed over in the FFMA thread layout
// to gemm_epilogue, run by the 256 consumer threads, with the ring as scratch.
//
// Tiles are numbered on a 1D order in which the column tile is the fast index: the CTAs running together cover a row
// tile's column tiles side by side, so its A rows come from HBM once and its other column tiles find them in L2.
// (Every layer's A is larger than the L2; with the row tile fast, A was read from HBM once per column tile.)
//   EPI_PLAIN and EPI_SEMCH are persistent (tc_persistent): min(tiles, SMs) CTAs, CTA i takes tiles i, i + grid, ...
//     The ring's stage counter c and the mbarrier phases run on across tiles (stage c of the CTA's run uses slot
//     c % STAGES; `full` is waited on parity (c / STAGES) & 1, `empty` before refilling on (c / STAGES - 1) & 1), and
//     the producer rebuilds its row table (`rowbase`, under named barrier 3 over its 128 threads) at each tile, so it
//     fills the next tile's first stages while the consumers finish the current one.  The consumers write a finished
//     tile into the staging buffer, meet at a named barrier (SemCH: two), and one of them issues the tensor stores; it
//     waits for the TMA engine to have read them only before the next tile is written there (and before it exits), so
//     the consumers go on to the next tile's K loop while the stores drain.
//   EPI_GLOBAL uses the ring as its epilogue's scratch, so it runs one tile per CTA (grid = tiles).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <vector>
#include "gast_common.cuh"
#include "gemm_ffma.cuh"

namespace gast {

// f16 == false (training's copies): hi and lo, for 3xTF32 and 1xTF32.  f16 == true (inference's copies): hi for
// 1xTF32 and the F16X3 pair h16 with its exponent s_W.
struct TcWeights {
  float* hi = nullptr;   // tf32(W), stored [K/4][N][4]
  float* lo = nullptr;   // tf32(W - tf32(W)), same layout; not allocated when f16
  __half* h16 = nullptr; // fp16(W 2^s_W) then fp16(W 2^s_W - hi), each stored [K/8][N][8]
  int* sw = nullptr;     // s_W (device)
  CUtensorMap map_hi, map_lo, map_h16hi, map_h16lo;
  int N = 0, K = 0;
  bool f16 = false;
  bool ready = false;
};

// precision of the core: TC_3XTF32 and TC_F16X3 are gast_set_precision's mode 0 (training and inference), TC_1XTF32
// its mode 1; TC_F16 is the half form (fp16 activations, gemm_tc_h_kernel)
enum { TC_3XTF32 = 0, TC_1XTF32 = 1, TC_F16X3 = 2, TC_F16 = 3 };

#ifndef GAST_TC1_STAGES
#define GAST_TC1_STAGES 3                             // ring depth of the 1xTF32 form: 4 and 5 measured no faster (DESIGN.md §4.1)
#endif
#ifndef GAST_TC16_STAGES
#define GAST_TC16_STAGES 3                            // ring depth of the F16X3 form: 4 measured within noise of 3 (DESIGN.md §4.1)
#endif

constexpr int TC_BM = 128, TC_BN = 128;
constexpr int TC_KS = 32;                            // K per ring stage; segment widths must be multiples of it
constexpr int TC_KP = 16;                            // K per partial sum, added into the tile sum with RN
constexpr int TC_THREADS = 384;                      // warpgroup 0 produces, warpgroups 1 and 2 consume
constexpr int TC_PRODUCER_REGS = 40, TC_CONSUMER_REGS = 232;   // 128 * 40 + 256 * 232 <= 64K registers of the SM
constexpr int TC_B_BYTES = TC_BN * TC_KS * 4;        // one of B_hi / B_lo in a stage
constexpr int TC_B16_BYTES = TC_BN * TC_KS * 2;      // the same in F16X3
// A stage: 128 dense rows of 32 floats (128 B) in TMA's 128-byte swizzle, 16-byte chunk c of row r at chunk
// c ^ (r & 7) (tc_achunk); 1024-byte aligned in every slot
constexpr int TC_A_BYTES = TC_BM * TC_KS * 4;
// B copy bytes, B copies per slot, slot size and ring depth of each precision
__host__ __device__ constexpr int tc_bbytes(int prec) { return prec == TC_F16X3 ? TC_B16_BYTES : TC_B_BYTES; }
__host__ __device__ constexpr int tc_nb(int prec) { return prec == TC_1XTF32 ? 1 : 2; }
__host__ __device__ constexpr int tc_slot(int prec) {                       // B_hi [| B_lo] | A
  return tc_nb(prec) * tc_bbytes(prec) + TC_A_BYTES;
}
__host__ __device__ constexpr int tc_stages(int prec) {
  return prec == TC_1XTF32 ? GAST_TC1_STAGES : prec == TC_F16X3 ? GAST_TC16_STAGES : 3;
}
__host__ __device__ constexpr int tc_ring(int prec) { return tc_stages(prec) * tc_slot(prec); }
constexpr int TC_STG_LD = 136;                       // [row][col] stride of the accumulator hand-over to the epilogue
constexpr int TC_ROWBASE_BYTES = 3 * 128 * sizeof(long long);
constexpr int TC_SMEM_MAX = 200 * 1024;              // the half form's bound
constexpr int TC_SMEM_OPTIN = 227 * 1024;            // the SM's opt-in shared memory per block: gemm_tc_kernel's bound
constexpr int TC_TILE_BYTES = TC_BM * TC_BN * 4;     // the persistent forms' staging buffer: one fp32 tile
// EPI_PLAIN and EPI_SEMCH run a persistent tile loop with a staging buffer of their own; EPI_GLOBAL, whose epilogue
// takes the ring as scratch, one tile per CTA
__host__ __device__ constexpr bool tc_persistent(int epi) { return epi == EPI_PLAIN || epi == EPI_SEMCH; }
static_assert(tc_slot(TC_3XTF32) % 1024 == 0 && tc_slot(TC_1XTF32) % 1024 == 0 && tc_slot(TC_F16X3) % 1024 == 0 &&
              TC_B16_BYTES % 1024 == 0, "ring slots and their A stages stay 1024-byte aligned");
static_assert(tc_ring(TC_1XTF32) + 16 * tc_stages(TC_1XTF32) + TC_ROWBASE_BYTES + 1024 <= TC_SMEM_MAX &&
              tc_ring(TC_F16X3) + 16 * tc_stages(TC_F16X3) + TC_ROWBASE_BYTES + 1024 <= TC_SMEM_MAX,
              "every ring fits the shared memory the core may use");

// rowbase | ring (1024-byte aligned) | persistent forms: staging buffer | a full and an empty mbarrier per slot |
// persistent forms: the residual's mbarrier
__host__ __device__ inline size_t tc_smem_bytes(int prec, int epi, int J, int fpt, int hpt) {
  if (tc_persistent(epi))
    return TC_ROWBASE_BYTES + 1024 + (size_t)tc_ring(prec) + TC_TILE_BYTES + 16 * tc_stages(prec) + 8;
  size_t m = (size_t)tc_ring(prec) + 16 * tc_stages(prec);
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
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y, int z,
                                            int w) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int x, int y) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(src), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int x, int y, int z) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(map), "r"(src), "r"(x), "r"(y), "r"(z) : "memory");
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

// float offset of 16-byte chunk c of row r in a 128-byte-swizzled [rows][32] fp32 stage
__device__ __forceinline__ int tc_achunk(int r, int c) { return r * TC_KS + ((c ^ (r & 7)) << 2); }

// An A segment whose frame map is affine over the whole launch: T_in == t_mul T_out, so map_frame(f) = t_mul f + t_off
// across clip boundaries, and tap k of output frame f, joint j, reads source row (t_mul f + t_off) J + j plus k
// tap_stride floats.  Its stages are TMA boxes of a 4D map (tc_encode_taps): identity segments (the 1x1 layers, SemCH,
// the attention GEMMs, the block concatenations), the strided stage convolutions and the taps of a stream's ring.
// Other segments (the dilated schedule across clips, the streams' chunk calls) are gathered per row by cp.async.
// tc_supported has already required Kc % 32 == 0 and tap strides of 16-byte multiples.
__host__ __device__ inline bool tc_map_affine(const RowMap& m) {
  return m.t_mul >= 1 && m.t_off >= 0 && m.T_in == m.t_mul * m.T_out;
}
__host__ __device__ inline bool tc_seg_tma(const ASeg& s) {
  return tc_map_affine(s.map) && (s.K == s.Kc || s.tap_stride > 0);
}
// The plain epilogue's residual by TMA (EPI_PLAIN): an affine residual map over a 16-byte-aligned residual with rows of
// 16-byte multiples.  Each tile's residual columns are then loaded into the staging buffer during the K loop
// (tc_load_res) instead of being read by __ldg after it.
__host__ __device__ inline bool tc_res_tma(const GemmP& p) {
  return p.res && tc_map_affine(p.res_map) && !(reinterpret_cast<uintptr_t>(p.res) & 15) && p.res_ld % 4 == 0;
}
// The half form's TMA segments: tile rows contiguous in the source (identity frame map, one tap), output row r of the
// tile starting at frame f0 at source row f0 J + r (tc_encode_a16)
__host__ __device__ inline bool tc_seg_tma_h(const ASeg& s) {
  return s.tap_stride == 0 && s.map.T_in == s.map.T_out && s.map.t_mul == 1 && s.map.t_off == 0;
}
// per A segment taken by tc_seg_tma: tc_encode_taps (tc_encode_a16 in the half form); out: the plain epilogue's
// output, fp32 {N, F J} at row stride ld_out, box {32, fpt J}, or the SemCH epilogue's (tc_encode_semch), 128-byte
// swizzle.  (gemm_tc_kernel's plain epilogue takes the residual's map, when tc_res_tma takes it, as a parameter of
// its own: tc_encode_taps of {N columns, one tap, res_map}.)
struct TcActMaps {
  CUtensorMap seg[3];
  CUtensorMap out;
};

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

// A fragment rows r0, r0 + 8 of the k8 steps s0, s0 + 1 of a slot's A (swizzled, tc_achunk), rounded to tf32 (hi)
// and, in 3xTF32, the rounding error split off as lo.  k = 8 s + t sits in chunk 2 s, k + 4 in chunk 2 s + 1; the
// warp's eight rows r0 & 7 = 0 .. 7 then spread each load over all 32 banks.
template <int PREC>
__device__ __forceinline__ void tc_load_a(const float* A, int r0, int t, int s0, uint32_t (&ah)[2][4],
                                          uint32_t (&al)[2][4]) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int c = 2 * (s0 + i);
    const float x[4] = {A[tc_achunk(r0, c) + t], A[tc_achunk(r0 + 8, c) + t], A[tc_achunk(r0, c + 1) + t],
                        A[tc_achunk(r0 + 8, c + 1) + t]};
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

// d (+)= a . B, m64n128k16, fp16 operands (A from registers, B K-major from shared memory), fp32 accumulate
__device__ __forceinline__ void wgmma_f16(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %68, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %69, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(scale_d), "l"(bdesc));
}

// One F16X3 16-K partial: d = A_lo.B_hi + A_hi.B_lo + A_hi.B_hi (small products first) of the k16 step s of the slot
// at sb, issued as one wgmma group
__device__ __forceinline__ void tc_partial16(float (&d)[64], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                             uint32_t sb, int s) {
  tile_fence(d);
  wgmma_fence();
  const uint64_t dh = tc_bdesc(sb + s * 4096), dl = tc_bdesc(sb + TC_B16_BYTES + s * 4096);
  wgmma_f16(d, al, dh, 0);
  wgmma_f16(d, ah, dl, 1);
  wgmma_f16(d, ah, dh, 1);
  wgmma_commit();
}

__device__ __forceinline__ float exp2i(int e) { return __int_as_float((e + 127) << 23); }   // 2^e, e in [-126, 127]

// s_r of a row whose max |a| is m: m 2^s_r in [2^14, 2^15) from m's exponent bits, 0 for m == 0 or not finite,
// clamped to [smin, smax] (tc_scale_bounds)
__device__ __forceinline__ int tc_row_exp(float m, int smin, int smax) {
  const int eb = __float_as_int(m) >> 23;                                // m >= 0: the biased exponent
  const int s = (m == 0.f || eb == 255) ? 0 : 141 - eb;                  // m in [2^(eb-127), 2^(eb-126))
  return min(max(s, smin), smax);
}

// s_r's range: 2^s_r and 2^-(s_r + s_W) both normal fp32
__device__ __forceinline__ void tc_scale_bounds(int sw, int& smin, int& smax) {
  smin = max(-126, -127 - sw);
  smax = min(127, 126 - sw);
}

// The F16X3 A fragments of both k16 steps of a slot's A (swizzled, tc_achunk): rows r0, r0 + 8 at k pairs
// 16 s + 2t and 16 s + 2t + 8, scaled per row by 2^s_r and split into fp16 hi / lo; u0, u1 = 2^-(s_r + s_W) of the
// two rows.  The quad's four threads hold a row's 32 values of the stage between them.  k = 16 s + 2t sits in chunk
// 4 s + t / 2 at float 2 (t & 1), k + 8 two chunks on; the swizzle spreads a warp's 64-bit loads over all 32 banks
// in the two wavefronts 256 bytes take.
__device__ __forceinline__ void tc_load_a16(const float* A, int r0, int t, int sw, int smin, int smax,
                                            uint32_t (&ah)[2][4], uint32_t (&al)[2][4], float& u0, float& u1) {
  float2 x[2][4];
  const int w = 2 * (t & 1);
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const int c = 4 * s + (t >> 1);
    x[s][0] = *reinterpret_cast<const float2*>(A + tc_achunk(r0, c) + w);
    x[s][1] = *reinterpret_cast<const float2*>(A + tc_achunk(r0 + 8, c) + w);
    x[s][2] = *reinterpret_cast<const float2*>(A + tc_achunk(r0, c + 2) + w);
    x[s][3] = *reinterpret_cast<const float2*>(A + tc_achunk(r0 + 8, c + 2) + w);
  }
  float m[2] = {0.f, 0.f};
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int q = 0; q < 4; ++q) m[q & 1] = fmaxf(m[q & 1], fmaxf(fabsf(x[s][q].x), fabsf(x[s][q].y)));
  float v[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
    m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
    const int e = tc_row_exp(m[h], smin, smax);
    v[h] = exp2i(e);
    (h ? u1 : u0) = exp2i(-(e + sw));
  }
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float2 y = make_float2(x[s][q].x * v[q & 1], x[s][q].y * v[q & 1]);
      const __half2 hi = __float22half2_rn(y);
      const float2 hf = __half22float2(hi);
      const __half2 lo = __float22half2_rn(make_float2(y.x - hf.x, y.y - hf.y));
      ah[s][q] = *reinterpret_cast<const uint32_t*>(&hi);
      al[s][q] = *reinterpret_cast<const uint32_t*>(&lo);
    }
}

// acc += 2^-(s_r + s_W) part, one rounding per element (the multiplier is a power of two); u0 scales the fragment's
// row r0, u1 its row r0 + 8
__device__ __forceinline__ void tc_add_scaled(float (&acc)[64], float (&part)[64], float u0, float u1) {
  tile_fence(part);
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = fmaf(part[i], (i & 2) ? u1 : u0, acc[i]);
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

// EPI_PLAIN on the consumers' wgmma fragments (rows r0, r0 + 8; columns 8 i + 2t, + 1 in acc[4 i ..]): bias, ReLU and
// residual in gemm_epilogue's order, so the bits are the same, then the tile goes through the staging buffer (`stage`,
// shared address sb) to TMA as four 128-byte-swizzled column blocks of 32 floats ([128][32] each, 16 KB apart), and
// consumer thread 0 stores them with `out` (tile rows f0 J .. f0 J + fpt J - 1 of the box; the map's dims drop rows
// past F J and columns past N).  res_stg: the residual is already in the buffer (tc_load_res, landed), each value at
// the position its output takes, and is read from there; otherwise it is read by __ldg.  The buffer must otherwise be
// free (the previous stores read) when this is called; the stores are committed as one bulk group, not waited for.
__device__ __forceinline__ void tc_store_plain(const GemmP& p, const float (&acc)[64], unsigned char* stage,
                                               uint32_t sb, const CUtensorMap& out, int r0, int t, int ct, int f0,
                                               int vrows, int n0, bool res_stg) {
  const int J = p.J;
  const float* resrow[2] = {nullptr, nullptr};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;
    if (p.res && !res_stg && r < vrows) {
      const int fr = r / J, j = r - fr * J;
      resrow[h] = p.res + (map_frame(p.res_map, f0 + fr) * J + j) * (long long)p.res_ld;
    }
  }
  float* S = reinterpret_cast<float*>(stage);
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int col = 8 * i + 2 * t, n = n0 + col;
    const bool in = n < p.N;                                            // N % 4 == 0: n + 1 < N too
    float2 b = make_float2(0.f, 0.f);
    if (p.bias && in) b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
      if (p.bias) { v0 += b.x; v1 += b.y; }
      if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      const int r = r0 + 8 * h;
      float2* o = reinterpret_cast<float2*>(S + (i >> 2) * (TC_BM * TC_KS) + tc_achunk(r, col >> 2 & 7) + (col & 3));
      if (resrow[h] && in) {
        const float2 rr = __ldg(reinterpret_cast<const float2*>(resrow[h] + n));
        v0 += rr.x; v1 += rr.y;
      } else if (res_stg) {                                             // the residual tc_load_res staged here
        const float2 rr = *o;
        v0 += rr.x; v1 += rr.y;
      }
      *o = make_float2(v0, v1);
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // the writes above, seen by the TMA engine
  epi_sync();
  if (ct == 0) {
    for (int cb = 0; cb < TC_BN / TC_KS && n0 + cb * TC_KS < p.N; ++cb)
      tma_store_2d(&out, sb + cb * TC_A_BYTES, n0 + cb * TC_KS, f0 * J);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
}

// EPI_SEMCH on the consumers' wgmma fragments.  The tile is 64 channels of one mask: columns 0 .. 63 hold the self
// products X.W0, columns 64 .. 127 the neighbour products H = X.W1 (gemm_epilogue).  The staging buffer (`stage`,
// shared address sb) holds four 128-byte-swizzled [128][32] float blocks (tc_achunk): blocks 0 and 1 take H, blocks 2
// and 3 the output O.  Every thread writes its H columns (acc[4 i ..], i >= 8), and after a barrier mixes its rows r0,
// r0 + 8 below vrows in its channel pairs c = chan0 + 8 i + 2t, + 1 (i < 8):  v = shift, then
// v = fmaf(coef[z][c], h_jj[c], v) over the row's neighbours z in row_ptr order, the self term from its own fragment
// and the others from H at their row of the same frame, then ReLU.  That is gemm_epilogue's order, so the bits are the
// same.  Consumer thread 0 then stores each 32-channel O block whose first channel is below C with `out`
// (tc_encode_semch: channels {C, masks, F J}, which drops channels past C of each mask and rows past F J).  The buffer
// must be free (the previous stores read) when this is called; the stores are committed as one bulk group, not waited
// for.
__device__ __forceinline__ void tc_store_semch(const GemmP& p, const float (&acc)[64], unsigned char* stage,
                                               uint32_t sb, const CUtensorMap& out, int r0, int t, int ct, int ctile,
                                               int f0, int vrows) {
  const int J = p.J, C = p.C;
  float* S = reinterpret_cast<float*>(stage);
#pragma unroll
  for (int i = 8; i < 16; ++i) {
    const int col = 8 * i + 2 * t - 64;
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(S + (col >> 5) * (TC_BM * TC_KS) + tc_achunk(r0 + 8 * h, col >> 2 & 7) + (col & 3)) =
          make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
  }
  epi_sync();
  const int mask = ctile / p.tiles_per_mask;
  const int chan0 = (ctile - mask * p.tiles_per_mask) * 64;
  const NbrTable& nb = p.nbr[mask];
  const float* coef = p.coef[mask] + chan0 + 2 * t;
  float2 sh[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    sh[i] = make_float2(0.f, 0.f);
    if (p.shift && chan0 + 8 * i + 2 * t < C)                           // C % 4 == 0: c + 1 < C too
      sh[i] = __ldg(reinterpret_cast<const float2*>(p.shift + mask * C + chan0 + 8 * i + 2 * t));
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;
    if (r >= vrows) continue;
    const int fr = r / J, ji = r - fr * J;
    float2 v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = sh[i];
    const int zend = nb.row_ptr[ji + 1];
    for (int z = nb.row_ptr[ji]; z < zend; ++z) {
      const int jj = nb.col[z];
      const float* cz = coef + (long long)z * C;
      const int hr = fr * J + jj;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int col = 8 * i + 2 * t;
        float2 cf = make_float2(0.f, 0.f);
        if (chan0 + col < C) cf = __ldg(reinterpret_cast<const float2*>(cz + 8 * i));
        float2 hv;
        if (jj == ji) hv = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        else hv = *reinterpret_cast<const float2*>(S + (i >> 2) * (TC_BM * TC_KS) + tc_achunk(hr, col >> 2 & 7) +
                                                   (col & 3));
        v[i].x = fmaf(cf.x, hv.x, v[i].x);
        v[i].y = fmaf(cf.y, hv.y, v[i].y);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int col = 8 * i + 2 * t;
      if (p.relu) { v[i].x = fmaxf(v[i].x, 0.f); v[i].y = fmaxf(v[i].y, 0.f); }
      *reinterpret_cast<float2*>(S + (2 + (i >> 2)) * (TC_BM * TC_KS) + tc_achunk(r, col >> 2 & 7) + (col & 3)) = v[i];
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // the writes above, seen by the TMA engine
  epi_sync();
  if (ct == 0) {
    for (int cb = 0; cb < 2 && chan0 + cb * TC_KS < C; ++cb)
      tma_store_3d(&out, sb + (2 + cb) * TC_A_BYTES, chan0 + cb * TC_KS, mask, f0 * J);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
  }
}

// consumer thread 0: wait until the TMA engine has read every tensor store it issued from the staging buffer
__device__ __forceinline__ void tc_stores_read(int ct) {
  if (ct == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// Whether this CTA has a tile after its tile u (tile blockIdx.x + u gridDim.x), and that tile's row and column tile.
// %ctaid and %nctaid are read with volatile moves, so that the consumers recompute the tile after their K loop instead
// of keeping it in registers through it.
__device__ __forceinline__ bool tc_tile_at(const GemmP& p, int u, int& rt, int& ctile) {
  uint32_t b, g;
  asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(b));
  asm volatile("mov.u32 %0, %%nctaid.x;" : "=r"(g));
  const int col_tiles = (p.N + TC_BN - 1) / TC_BN;
  const long long tile = b + (long long)u * g;
  if (tile >= (long long)((p.F + p.fpt - 1) / p.fpt) * col_tiles) return false;
  rt = (int)(tile / col_tiles);
  ctile = (int)(tile - (long long)rt * col_tiles);
  return true;
}

// Consumer thread 0, in the K loop of the CTA's tile u: once the TMA engine has read the previous tile's stores from
// the staging buffer (at `stg`), load the tile's residual rows into it, one box of `map` per 32-column block below N,
// on the mbarrier `bar` (completed once per tile; tc_store_plain waits on parity u & 1).  Each block lands in the
// swizzled [128][32] layout tc_store_plain writes the output in, so every consumer thread finds its residual values
// at the positions it then overwrites.
__device__ __forceinline__ void tc_load_res(const GemmP& p, const CUtensorMap& map, uint32_t stg, uint32_t bar, int u) {
  int rt, ctile;
  tc_tile_at(p, u, rt, ctile);
  const int n0 = ctile * TC_BN, f0 = rt * p.fpt;
  const int nb = min(TC_BN / TC_KS, (p.N - n0 + TC_KS - 1) / TC_KS);
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  mbar_arrive_expect_tx(bar, nb * TC_KS * 4 * p.J * p.fpt);
  for (int cb = 0; cb < nb; ++cb) tma_load_4d(stg + cb * TC_A_BYTES, &map, bar, n0 + cb * TC_KS, 0, 0, f0);
}

// mlo is not read in 1xTF32, sw (s_W) only in F16X3, am.seg[s] only for the segments tc_seg_tma takes, am.out only in
// EPI_PLAIN and EPI_SEMCH, mres only in EPI_PLAIN when tc_res_tma takes the residual
template <int EPI, int PREC>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ GemmP p, const __grid_constant__ CUtensorMap mhi,
               const __grid_constant__ CUtensorMap mlo, const __grid_constant__ TcActMaps am,
               const int* __restrict__ sw, const __grid_constant__ CUtensorMap mres) {
  constexpr int STAGES = tc_stages(PREC), SLOT = tc_slot(PREC), NB = tc_nb(PREC);
  constexpr int BBYTES = tc_bbytes(PREC);
  constexpr int KSH = PREC == TC_F16X3 ? 3 : 2;                         // log2 of the k's per 16-byte row of a B copy
  constexpr int STG = tc_persistent(EPI) ? TC_TILE_BYTES : 0;
  // the plain epilogue's residual by TMA (tc_load_res), in the inference forms; 3xTF32 (training and the gradients)
  // keeps its K loop as it was and reads the residual by __ldg
  constexpr bool RES_TMA = EPI == EPI_PLAIN && PREC != TC_3XTF32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  long long* rowbase = reinterpret_cast<long long*>(smem_raw);          // [3][128]
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t rb = (raw + TC_ROWBASE_BYTES + 1023) & ~1023u;        // ring base (shared address)
  unsigned char* ring = smem_raw + (rb - raw);
  const uint32_t stg = rb + tc_ring(PREC);                              // persistent forms: staging buffer
  const uint32_t full0 = stg + STG;                                     // per ring slot: stage landed
  const uint32_t empty0 = full0 + 8 * STAGES;                           // per ring slot: both consumers done with it
  const uint32_t resbar = empty0 + 8 * STAGES;                          // EPI_PLAIN: the tile's residual landed

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int J = p.J;
  int tma_segs = 0;                                                     // bit s: segment s is loaded by TMA
  for (int s = 0; s < p.nseg; ++s) tma_segs |= tc_seg_tma(p.seg[s]) << s;
  const bool gather = tma_segs != (1 << p.nseg) - 1;                    // some segment is gathered per row
  const uint32_t abytes = TC_KS * 4 * J * p.fpt;                        // a TMA segment's stage: the tile's fpt J rows

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, gather ? 1 + 128 : 1);
      mbar_init(empty0 + 8 * s, 8);
    }
    if (RES_TMA) mbar_init(resbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  int nstages = 0;
  for (int s = 0; s < p.nseg; ++s) nstages += p.seg[s].K / TC_KS;

  if (warp < 4) {
    // producer: stage c of the CTA's run into ring slot c % STAGES once both consumers have released the slot's
    // previous stage
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (!gather && tid != 0) return;                                    // the elected thread issues every stage
    const int q = tid & 7, rq = tid >> 3;                               // k-quad q of rows rq + 16 i
    const uint32_t adst = NB * BBYTES + 4 * tc_achunk(rq, q);           // its slot offset in row rq; rows + 16 i follow
    const int col_tiles = (p.N + TC_BN - 1) / TC_BN;
    const int tiles = ((p.F + p.fpt - 1) / p.fpt) * col_tiles;
    int c = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      const int rt = tile / col_tiles;
      const int f0 = rt * p.fpt, n0 = (tile - rt * col_tiles) * TC_BN;
      if (gather) {                                                     // the tile's row table, for the gathered rows
        const int vrows = min(p.fpt, p.F - f0) * J;
        asm volatile("bar.sync 3, 128;" ::: "memory");                  // every thread has issued the last tile
        for (int i = tid; i < p.nseg * 128; i += 128) {
          const int s = i >> 7, r = i & 127;
          long long off = -1;
          if (r < vrows) {
            const int fr = r / J, j = r - fr * J;
            off = (map_frame(p.seg[s].map, f0 + fr) * J + j) * (long long)p.seg[s].ld;
          }
          rowbase[i] = off;
        }
        asm volatile("bar.sync 3, 128;" ::: "memory");
      }
      int seg = 0, k0 = 0, kcol = 0, tap = 0, kin = 0;                  // stage start: segment, K in it, W column, tap
      for (int k = 0; k < nstages; ++k, ++c) {
        const int slot = c % STAGES;
        if (c >= STAGES) mbar_wait(empty0 + 8 * slot, (c / STAGES - 1) & 1);
        const uint32_t sb = rb + slot * SLOT, full = full0 + 8 * slot;
        const bool tma_a = (tma_segs >> seg) & 1;
        if (tid == 0) {
          mbar_arrive_expect_tx(full, NB * BBYTES + (tma_a ? abytes : 0));
          const int kq = (kcol + k0) >> KSH;
          tma_load_2d(sb, &mhi, full, 2 * n0, kq);
          if (NB == 2) tma_load_2d(sb + BBYTES, &mlo, full, 2 * n0, kq);
          if (tma_a) tma_load_4d(sb + NB * BBYTES, &am.seg[seg], full, kin, 0, tap, f0);
        }
        const ASeg& sg = p.seg[seg];
        if (tma_a) {
          if (gather) mbar_arrive(full);                                // the barrier counts 128 producer arrivals
        } else {
          const float* src = sg.base + tap * sg.tap_stride + kin + q * 4;
#pragma unroll
          for (int i = 0; i < TC_BM / 16; ++i) {
            const long long off = rowbase[seg * 128 + rq + 16 * i];
            cp_async16(sb + adst + i * 16 * 128, off >= 0 ? src + off : sg.base, off >= 0 ? 16 : 0);
          }
          cp_async_arrive(full);
        }
        k0 += TC_KS;
        kin += TC_KS;
        if (kin == sg.Kc) { kin = 0; ++tap; }
        if (k0 == sg.K) { kcol += sg.K; k0 = 0; tap = 0; ++seg; }
      }
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
  int s_w = 0, smin = 0, smax = 0;                                      // F16X3: s_W and s_r's range
  if constexpr (PREC == TC_F16X3) {
    s_w = *sw;
    tc_scale_bounds(s_w, smin, smax);
  }
  // The stage counter c is the only tile state carried through the K loop: the CTA's tile u is c / nstages - 1 after
  // it, and the tile itself is read again from the grid position (tc_tile_at).
  int c = 0;
  for (;;) {
    float acc[64], part0[64], part1[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const int cend = c + nstages;
    // EPI_PLAIN with tc_res_tma: consumer thread 0 loads the tile's residual after the tile's third stage (its last,
    // if it has fewer), when the last tile's stores have long been read and most of the K loop is left to hide it

    if constexpr (PREC == TC_F16X3) {
      for (; c < cend; ++c) {
        const int slot = c % STAGES;
        mbar_wait(full0 + 8 * slot, (c / STAGES) & 1);
        const uint32_t sb = rb + slot * SLOT;
        const float* A = reinterpret_cast<const float*>(ring + slot * SLOT + NB * BBYTES);
        uint32_t ah[2][4], al[2][4];
        float u0, u1;
        tc_load_a16(A, r0, t, s_w, smin, smax, ah, al, u0, u1);   // one scale per row and stage
        tc_partial16(part0, ah[0], al[0], sb, 0);
        tc_partial16(part1, ah[1], al[1], sb, 1);
        wgmma_wait<1>();
        tc_add_scaled(acc, part0, u0, u1);
        wgmma_wait<0>();
        tc_add_scaled(acc, part1, u0, u1);
        if (lane == 0) mbar_arrive(empty0 + 8 * slot);
        if (RES_TMA && ct == 0 && c + nstages - cend == min(2, nstages - 1) && tc_res_tma(p))
          tc_load_res(p, mres, stg, resbar, c / nstages);
      }
    } else {
      for (; c < cend; ++c) {
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
        if (RES_TMA && ct == 0 && c + nstages - cend == min(2, nstages - 1) && tc_res_tma(p))
          tc_load_res(p, mres, stg, resbar, c / nstages);
      }
    }
    int rt, ctile;
    const int u = c / nstages - 1;
    tc_tile_at(p, u, rt, ctile);
    const int fe = rt * p.fpt, nfe = min(p.fpt, p.F - fe);

    if constexpr (EPI == EPI_PLAIN) {
      tc_stores_read(ct);                       // the staging buffer is free once the last tile's stores are read
      epi_sync();
      const bool res_stg = RES_TMA && tc_res_tma(p);
      if (res_stg) mbar_wait(resbar, u & 1);   // the tile's residual, loaded into the buffer by tc_load_res
      tc_store_plain(p, acc, ring + tc_ring(PREC), stg, am.out, r0, t, ct, fe, nfe * J, ctile * TC_BN, res_stg);
      if (!tc_tile_at(p, u + 1, rt, ctile)) {
        tc_stores_read(ct);                     // the staging buffer stays until the engine has read it
        return;
      }
    } else if constexpr (EPI == EPI_SEMCH) {
      tc_stores_read(ct);                       // as EPI_PLAIN; tc_store_semch's first barrier follows
      tc_store_semch(p, acc, ring + tc_ring(PREC), stg, am.out, r0, t, ct, ctile, fe, nfe * J);
      if (!tc_tile_at(p, u + 1, rt, ctile)) {
        tc_stores_read(ct);
        return;
      }
    } else {
      epi_sync();                               // both consumers are done with the ring
      // hand the tile over in the FFMA thread layout gemm_epilogue<EPI_GLOBAL> expects
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
        const float4 a = *reinterpret_cast<const float4*>(S + r * TC_STG_LD + tx * 4);
        const float4 b = *reinterpret_cast<const float4*>(S + r * TC_STG_LD + 64 + tx * 4);
        out[i][0] = a.x; out[i][1] = a.y; out[i][2] = a.z; out[i][3] = a.w;
        out[i][4] = b.x; out[i][5] = b.y; out[i][6] = b.z; out[i][7] = b.w;
      }
      epi_sync();
      gemm_epilogue<EPI>(p, out, reinterpret_cast<float*>(ring), ct, fe, nfe, nfe * J, ctile * TC_BN, ctile);
      return;                                   // one tile per CTA (tc_persistent)
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// TC_F16, the half form (gast_set_activation_dtype(h, GAST_F16)): A and the output are fp16 in memory, so a MAC is one
// fp16 product,  D = 2^-s_W (A . fp16(W 2^s_W)),  with fp32 accumulation.  B is the F16X3 hi copy unchanged; the weight
// scale is applied once, to the finished tile, before the epilogue (a power of two: no rounding).  Both operands are
// read by wgmma from shared memory through descriptors (m64n128k16, SS form), in one layout: the no-swizzle K-major
// core-matrix layout of the B copies, [K/8][rows][8] halves (8 rows x 16 B core matrices, 128 B apart along the rows,
// 2048 B apart along K), so tc_bdesc describes A as well.  A stage is 128 rows x 32 K = 8 KB:
//   identity segments (tc_seg_tma_h): one 3D TMA box {8 halves, 128 rows, 4 k-octets} of a map with dims
//     {8, rows, Kc / 8} and strides {ld, 8} halves (tc_encode_a16), which lands in exactly that layout;
//   gathered segments: cp.async of 16 B = one row's k-octet, zero-filled outside the tile.
// K is chained in the accumulator: the tensor core's truncation bias (~0.5 ulp of fp32 per k16 MMA) stays far below
// the 2^-11 rounding of the fp16 operands (K = 1536 is 96 MMAs), so the two-level partial sums of the fp32-grade forms
// buy nothing here.  It runs one tile per CTA; tiles, ring protocol and producer are gemm_tc_kernel's; the epilogues
// read the residual and write the output as fp16 (tc_store_plain_h's TMA store of two [128][64]-half column blocks; SemCH through
// gemm_epilogue<EPI_SEMCH, __half>).  There is no EPI_GLOBAL form: a half model's attention mix is its own kernel
// (global_mix_kernel, J <= MIX_JMAX, which gast_set_activation_dtype requires).
#ifndef GAST_TCH_STAGES
#define GAST_TCH_STAGES 6
#endif
constexpr int TCH_STAGES = GAST_TCH_STAGES;
constexpr int TC_H_A_BYTES = TC_BM * TC_KS * 2;
constexpr int TC_H_SLOT = TC_B16_BYTES + TC_H_A_BYTES;
constexpr int TC_H_RING = TCH_STAGES * TC_H_SLOT;
static_assert(TC_H_SLOT % 1024 == 0 && TC_H_RING >= 2 * TC_BM * 64 * 2,
              "slots stay 1024-byte aligned, and the ring holds the plain epilogue's fp16 tile");

__host__ __device__ inline size_t tch_smem_bytes(int epi, int J, int fpt, int hpt) {
  size_t m = (size_t)TC_H_RING + 16 * TCH_STAGES;
  const size_t stg = (size_t)TC_BM * TC_STG_LD * 4;
  const size_t e = ffma_smem_bytes(epi, J, fpt, hpt) - TC_ROWBASE_BYTES;
  if (stg > m) m = stg;
  if (e > m) m = e;
  return TC_ROWBASE_BYTES + 1024 + m;
}

__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y, int z) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y), "r"(z) : "memory");
}

// d (+)= A . B, m64n128k16, fp16 operands both K-major in shared memory, fp32 accumulate; scale_d == 0 overwrites d
__device__ __forceinline__ void wgmma_f16ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, int scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(scale_d));
}

// EPI_PLAIN of the half form: tc_store_plain's order (bias, ReLU, residual read as fp16), each value rounded once to
// fp16, staged in the free ring as two 128-byte-swizzled [128][64]-half column blocks (16 KB apart) and stored with
// `out` (fp16 {N, F J}, box {64, fpt J}).
__device__ __forceinline__ void tc_store_plain_h(const GemmP& p, const float (&acc)[64], unsigned char* ring,
                                                 uint32_t rb, const CUtensorMap& out, int r0, int t, int ct, int f0,
                                                 int vrows, int n0) {
  const int J = p.J;
  const __half* resrow[2] = {nullptr, nullptr};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;
    if (p.res && r < vrows) {
      const int fr = r / J, j = r - fr * J;
      resrow[h] = reinterpret_cast<const __half*>(p.res) + (map_frame(p.res_map, f0 + fr) * J + j) * (long long)p.res_ld;
    }
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int col = 8 * i + 2 * t, n = n0 + col;
    const bool in = n < p.N;                                            // N % 4 == 0: n + 1 < N too
    float2 b = make_float2(0.f, 0.f);
    if (p.bias && in) b = __ldg(reinterpret_cast<const float2*>(p.bias + n));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float v0 = acc[4 * i + 2 * h], v1 = acc[4 * i + 2 * h + 1];
      if (p.bias) { v0 += b.x; v1 += b.y; }
      if (p.relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      if (resrow[h] && in) {
        const float2 rr = __half22float2(__ldg(reinterpret_cast<const __half2*>(resrow[h] + n)));
        v0 += rr.x; v1 += rr.y;
      }
      const int r = r0 + 8 * h;
      *reinterpret_cast<__half2*>(ring + (col >> 6) * (TC_BM * 128) + r * 128 + ((((col >> 3) & 7) ^ (r & 7)) << 4) +
                                  (col & 7) * 2) = __floats2half2_rn(v0, v1);
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");        // the writes above, seen by the TMA engine
  epi_sync();
  if (ct == 0) {
    for (int cb = 0; cb < 2 && n0 + cb * 64 < p.N; ++cb) tma_store_2d(&out, rb + cb * TC_BM * 128, n0 + cb * 64, f0 * J);
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  }
}

// The half form of gemm_tc_kernel: p's segment bases, out and res point to __half; lds, tap strides and residual
// strides count halves.  mb: the F16X3 hi copy's map; am.seg[s] (tc_encode_a16) for the segments tc_seg_tma_h takes,
// am.out (fp16, tc_encode_rows16) in EPI_PLAIN.
template <int EPI>   // EPI_PLAIN or EPI_SEMCH
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_h_kernel(const __grid_constant__ GemmP p, const __grid_constant__ CUtensorMap mb,
                 const __grid_constant__ TcActMaps am, const int* __restrict__ sw) {
  constexpr int STAGES = TCH_STAGES, SLOT = TC_H_SLOT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  long long* rowbase = reinterpret_cast<long long*>(smem_raw);          // [3][128]
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t rb = (raw + TC_ROWBASE_BYTES + 1023) & ~1023u;        // ring base (shared address)
  unsigned char* ring = smem_raw + (rb - raw);
  const uint32_t full0 = rb + TC_H_RING;
  const uint32_t empty0 = full0 + 8 * STAGES;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int J = p.J;
  int rt, ctile;
  tc_tile(p, rt, ctile);
  const int f0 = rt * p.fpt;
  const int nf = min(p.fpt, p.F - f0);
  const int vrows = nf * J;
  const int n0 = ctile * TC_BN;
  int tma_segs = 0;
  for (int s = 0; s < p.nseg; ++s) tma_segs |= tc_seg_tma_h(p.seg[s]) << s;
  const bool gather = tma_segs != (1 << p.nseg) - 1;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full0 + 8 * s, gather ? 1 + 128 : 1);
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
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (!gather && tid != 0) return;
    const int q = tid & 3, rq = tid >> 2;                               // k-octet q of rows rq + 32 i
    const uint32_t adst = TC_B16_BYTES + q * 2048 + rq * 16;
    const int row0 = f0 * J;
    int seg = 0, k0 = 0, kcol = 0, tap = 0, kin = 0;
    for (int c = 0; c < nstages; ++c) {
      const int slot = c % STAGES;
      if (c >= STAGES) mbar_wait(empty0 + 8 * slot, (c / STAGES - 1) & 1);
      const uint32_t sb = rb + slot * SLOT, full = full0 + 8 * slot;
      const bool tma_a = (tma_segs >> seg) & 1;
      if (tid == 0) {
        mbar_arrive_expect_tx(full, TC_B16_BYTES + (tma_a ? TC_H_A_BYTES : 0));
        tma_load_2d(sb, &mb, full, 2 * n0, (kcol + k0) >> 3);
        if (tma_a) tma_load_3d(sb + TC_B16_BYTES, &am.seg[seg], full, 0, row0, kin >> 3);
      }
      const ASeg& sg = p.seg[seg];
      if (tma_a) {
        if (gather) mbar_arrive(full);
      } else {
        const __half* base = reinterpret_cast<const __half*>(sg.base);
        const __half* src = base + tap * sg.tap_stride + kin + q * 8;
#pragma unroll
        for (int i = 0; i < TC_BM / 32; ++i) {
          const long long off = rowbase[seg * 128 + rq + 32 * i];
          cp_async16(sb + adst + i * 32 * 16, off >= 0 ? src + off : base, off >= 0 ? 16 : 0);
        }
        cp_async_arrive(full);
      }
      k0 += TC_KS;
      kin += TC_KS;
      if (kin == sg.Kc) { kin = 0; ++tap; }
      if (k0 == sg.K) { kcol += sg.K; k0 = 0; tap = 0; ++seg; }
    }
    cp_async_wait_all();
    return;
  }

  // consumers: warpgroup 1 + w multiplies rows 64 w .. 64 w + 63 (1024 B into each octet plane of the A stage)
  setmaxnreg_inc<TC_CONSUMER_REGS>();
  const int ct = tid - 128;
  const int wg = ct >> 7, wq = (ct >> 5) & 3;
  const int g = lane >> 2, t = lane & 3;
  const int r0 = wg * 64 + wq * 16 + g;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  for (int c = 0; c < nstages; ++c) {
    const int slot = c % STAGES;
    mbar_wait(full0 + 8 * slot, (c / STAGES) & 1);
    const uint32_t sb = rb + slot * SLOT, sa = sb + TC_B16_BYTES + wg * 1024;
    tile_fence(acc);
    wgmma_fence();
    wgmma_f16ss(acc, tc_bdesc(sa), tc_bdesc(sb), c > 0);
    wgmma_f16ss(acc, tc_bdesc(sa + 4096), tc_bdesc(sb + 4096), 1);
    wgmma_commit();
    wgmma_wait<0>();
    tile_fence(acc);
    if (lane == 0) mbar_arrive(empty0 + 8 * slot);
  }
  const float u = exp2i(-*sw);                                          // 2^-s_W
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] *= u;
  epi_sync();
  tc_tile(p, rt, ctile);
  const int fe = rt * p.fpt, nfe = min(p.fpt, p.F - fe);

  if constexpr (EPI == EPI_PLAIN) {
    tc_store_plain_h(p, acc, ring, rb, am.out, r0, t, ct, fe, nfe * J, ctile * TC_BN);
    return;
  }
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
    const float4 a = *reinterpret_cast<const float4*>(S + r * TC_STG_LD + tx * 4);
    const float4 b = *reinterpret_cast<const float4*>(S + r * TC_STG_LD + 64 + tx * 4);
    out[i][0] = a.x; out[i][1] = a.y; out[i][2] = a.z; out[i][3] = a.w;
    out[i][4] = b.x; out[i][5] = b.y; out[i][6] = b.z; out[i][7] = b.w;
  }
  epi_sync();
  gemm_epilogue<EPI, __half>(p, out, reinterpret_cast<float*>(ring), ct, fe, nfe, nfe * J, ctile * TC_BN, ctile);
}

// W [N][K] -> hi / lo in the TMA-friendly layout [K/4][N][4] (both TF32 forms read hi = tf32(W)); lo may be null
__global__ void tc_split_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int N, int K) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * K) return;
  const int n = (int)(i / K), k = (int)(i - (long long)n * K);
  const float x = w[i];
  const float h = __uint_as_float(tf32_bits(x));
  const long long o = ((long long)(k >> 2) * N + n) * 4 + (k & 3);
  hi[o] = h;
  if (lo) lo[o] = __uint_as_float(tf32_bits(x - h));
}

// s_W of W [n]: max |W| 2^s_W in [2^14, 2^15), 0 for an all-zero or non-finite W.  One block.
__global__ void tc_wscale_kernel(const float* __restrict__ w, long long n, int* __restrict__ sw) {
  __shared__ float red[32];
  float m = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, fabsf(w[i]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (threadIdx.x == 0) *sw = (m == 0.f || !isfinite(m)) ? 0 : 14 - ilogbf(m);   // ilogbf: subnormals too
  }
}

// W [N][K] -> fp16(W 2^s_W) and fp16(W 2^s_W - hi), each in the TMA-friendly layout [K/8][N][8]
__global__ void tc_split16_kernel(const float* __restrict__ w, const int* __restrict__ sw, __half* __restrict__ hi,
                                  __half* __restrict__ lo, int N, int K) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)N * K) return;
  const int n = (int)(i / K), k = (int)(i - (long long)n * K);
  const float x = scalbnf(w[i], *sw);
  const __half h = __float2half_rn(x);
  const long long o = ((long long)(k >> 3) * N + n) * 8 + (k & 7);
  hi[o] = h;
  lo[o] = __float2half_rn(x - __half2float(h));
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

// fp32 [rows][cols] at row stride ld floats, box {32, box_rows} (128-byte rows), 128-byte swizzle; reads past the
// dims fill zeros, writes past them are dropped
inline int tc_encode_rows(CUtensorMap* m, const float* base, int cols, long long rows, int ld, int box_rows) {
  tc_encode_fn enc = tc_get_encode();
  if (!enc) return -1;
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)TC_KS, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -1;
}

// An A segment taken by tc_seg_tma as the stages of F output frames of J joints read it: fp32 dims {Kc, J, taps, F}
// with byte strides {ld, tap_stride, t_mul J ld} x 4 from base + t_off J ld, box {32, J, 1, fpt}, 128-byte swizzle.
// The box at (kin, 0, tap, f0) is the tile's fpt J rows of one stage, dense from the slot's 1024-byte-aligned A in the
// swizzle tc_achunk reads (chunk c of slot row r at c ^ (r & 7)); frames past F read as zeros, and slot rows past fpt J,
// which belong to no stored output row, keep what they held.  One tap: the tap stride is never used, and is given as
// a frame's J ld so that the strides stay nested.
inline int tc_encode_taps(CUtensorMap* m, const ASeg& s, int F, int J, int fpt) {
  tc_encode_fn enc = tc_get_encode();
  if (!enc) return -1;
  const int taps = s.K / s.Kc;
  const cuuint64_t row = (cuuint64_t)s.ld * 4, frame = (cuuint64_t)J * row;
  const cuuint64_t dims[4] = {(cuuint64_t)s.Kc, (cuuint64_t)J, (cuuint64_t)taps, (cuuint64_t)F};
  const cuuint64_t strides[3] = {row, taps > 1 ? (cuuint64_t)s.tap_stride * 4 : frame, (cuuint64_t)s.map.t_mul * frame};
  const cuuint32_t box[4] = {(cuuint32_t)TC_KS, (cuuint32_t)J, 1, (cuuint32_t)fpt};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const float* base = s.base + (long long)s.map.t_off * J * s.ld;
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -1;
}

// The SemCH epilogue's output: fp32 [rows][masks][C] at row stride ld floats (mask m's channels at column m C), as 3D
// {C, masks, rows}, box {32, 1, box_rows}, 128-byte swizzle, so a block's channels past C of its mask are dropped
// rather than written into the next mask's columns (C % 4 == 0 and ld % 4 == 0 keep the strides in 16-byte units)
inline int tc_encode_semch(CUtensorMap* m, const float* base, int C, int masks, long long rows, int ld, int box_rows) {
  tc_encode_fn enc = tc_get_encode();
  if (!enc) return -1;
  const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)masks, (cuuint64_t)rows};
  const cuuint64_t strides[2] = {(cuuint64_t)C * 4, (cuuint64_t)ld * 4};
  const cuuint32_t box[3] = {(cuuint32_t)TC_KS, 1, (cuuint32_t)box_rows};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -1;
}

// fp16 [rows][cols] at row stride ld halves, box {64, box_rows} (128-byte rows), 128-byte swizzle: the half form's
// plain-epilogue output
inline int tc_encode_rows16(CUtensorMap* m, const void* base, int cols, long long rows, int ld, int box_rows) {
  tc_encode_fn enc = tc_get_encode();
  if (!enc) return -1;
  const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -1;
}

// An fp16 A segment [rows][Kc] at row stride ld halves as the half form's stages read it: dims {8, rows, Kc / 8},
// strides {ld, 8} halves, box {8, 128, 4}, no swizzle, so a box lands as [4 k-octets][128 rows][8 halves]; rows past
// the end read as zeros
inline int tc_encode_a16(CUtensorMap* m, const void* base, int Kc, long long rows, int ld) {
  tc_encode_fn enc = tc_get_encode();
  if (!enc) return -1;
  const cuuint64_t dims[3] = {8, (cuuint64_t)rows, (cuuint64_t)(Kc / 8)};
  const cuuint64_t strides[2] = {(cuuint64_t)ld * 2, 16};
  const cuuint32_t box[3] = {8, (cuuint32_t)TC_BM, (cuuint32_t)(TC_KS / 8)};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -1;
}

// W: [N][K] fp32 K-major (device).  Allocates the copies once per shape and form, encodes their TMA maps and splits W
// into them: f16 == false, tf32 hi / lo (training: 3xTF32); f16 == true, tf32 hi (1xTF32) and the F16X3 pair with
// s_W (inference).  Returns 0 on success (t.ready says whether the core takes the shape), a cudaError_t or -1
// otherwise.
inline int tc_prepare_weights(TcWeights& t, const float* W, int N, int K, cudaStream_t st, std::vector<void*>* owned,
                              bool f16) {
  t.ready = false;
  if (K % TC_KS != 0 || N % 4 != 0) return 0;            // shape not taken by this core (FFMA runs it)
  if (!t.hi || t.N != N || t.K != K || t.f16 != f16) {
    tc_encode_fn enc = tc_get_encode();
    if (!enc) return -1;
    void* a = nullptr; void* b = nullptr;
    const size_t nb = f16 ? sizeof(__half) * 2 * (size_t)N * K + 256 : sizeof(float) * (size_t)N * K;
    cudaError_t e = cudaMalloc(&a, sizeof(float) * (size_t)N * K);
    if (e != cudaSuccess) return (int)e;
    e = cudaMalloc(&b, nb);
    if (e != cudaSuccess) { cudaFree(a); return (int)e; }
    owned->push_back(a); owned->push_back(b);
    t.hi = (float*)a; t.N = N; t.K = K; t.f16 = f16;
    t.lo = f16 ? nullptr : (float*)b;
    t.h16 = f16 ? (__half*)b : nullptr;
    t.sw = f16 ? (int*)(t.h16 + 2 * (size_t)N * K) : nullptr;
    // Each k-quad ([K/4][N][4] floats) or k-octet ([K/8][N][8] halves) row of a copy is N 16-byte pieces, contiguous,
    // so a copy is described as 2D of 8-byte elements: dims {2N, K/4 or K/8}, box {256, TC_KS/4 or TC_KS/8}.  A box is
    // then 8 (4) rows of 2 KB, the slot image of 128 n by 32 k, and the TMA engine issues 2 KB rows instead of
    // 16-byte ones.  Elements past 2N (columns past N of a partial last column tile) read as zero.
    cuuint64_t strides[1] = {(cuuint64_t)N * 16};
    cuuint32_t estr[2] = {1, 1};
    cuuint64_t dims[2] = {2 * (cuuint64_t)N, (cuuint64_t)(K / 4)};
    cuuint32_t box[2] = {2 * (cuuint32_t)TC_BN, (cuuint32_t)(TC_KS / 4)};
    for (int m = 0; m < (f16 ? 1 : 2); ++m) {
      CUresult r = enc(m ? &t.map_lo : &t.map_hi, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, m ? t.lo : t.hi, dims, strides, box,
                       estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                       CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { t.hi = nullptr; return -1; }
    }
    if (f16) {
      cuuint64_t d16[2] = {2 * (cuuint64_t)N, (cuuint64_t)(K / 8)};
      cuuint32_t b16[2] = {2 * (cuuint32_t)TC_BN, (cuuint32_t)(TC_KS / 8)};
      for (int m = 0; m < 2; ++m) {
        CUresult r = enc(m ? &t.map_h16lo : &t.map_h16hi, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, t.h16 + (size_t)m * N * K,
                         d16, strides, b16, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { t.hi = nullptr; return -1; }
      }
    }
  }
  const long long n = (long long)N * K;
  tc_split_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, t.hi, t.lo, N, K);
  if (f16) {
    tc_wscale_kernel<<<1, 1024, 0, st>>>(W, n, t.sw);
    tc_split16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(W, t.sw, t.h16, t.h16 + n, N, K);
  }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return (int)e;
  t.ready = true;
  return 0;
}

// The shapes the core takes are the same in every precision (each ring is no larger than the bound below).
inline bool tc_supported(const GemmP& p, int epi, const TcWeights& t) {
  if (!t.ready || t.K != p.ldw || t.N < p.N || p.N % 4) return false;
  // the plain and SemCH epilogues' tensor stores: the output map needs a 16-byte-aligned base and strides of 16-byte
  // units (SemCH's mask stride is C floats)
  if ((reinterpret_cast<uintptr_t>(p.out) & 15) || p.ld_out % 4) return false;
  if (epi == EPI_SEMCH && (p.C % 4 || p.tiles_per_mask <= 0 || p.N % (TC_BN * p.tiles_per_mask))) return false;
  for (int s = 0; s < p.nseg; ++s) {
    const ASeg& sg = p.seg[s];
    if (sg.K % TC_KS || sg.Kc % TC_KS || sg.ld % 4 || sg.tap_stride % 4) return false;
    if (reinterpret_cast<uintptr_t>(sg.base) & 15) return false;
  }
  const int hpt = epi == EPI_GLOBAL ? (p.heads < 4 ? p.heads : 4) : 1;
  if (tc_smem_bytes(TC_3XTF32, epi, p.J, p.fpt, hpt) > TC_SMEM_OPTIN) return false;
  if (tc_smem_bytes(TC_1XTF32, epi, p.J, p.fpt, hpt) > TC_SMEM_OPTIN) return false;
  if (tc_smem_bytes(TC_F16X3, epi, p.J, p.fpt, hpt) > TC_SMEM_OPTIN) return false;
  return true;
}

// The shapes the half form takes: fp16 copies, and every fp16 operand 16-byte aligned with 16-byte row strides
inline bool tc_supported_h(const GemmP& p, int epi, const TcWeights& t) {
  if (!t.ready || !t.f16 || t.K != p.ldw || t.N < p.N || p.N % 4) return false;
  if ((reinterpret_cast<uintptr_t>(p.out) & 15) || p.ld_out % 8) return false;
  if (p.res && (p.res_ld % 2 || (reinterpret_cast<uintptr_t>(p.res) & 3))) return false;
  for (int s = 0; s < p.nseg; ++s) {
    const ASeg& sg = p.seg[s];
    if (sg.K % TC_KS || sg.Kc % TC_KS || sg.ld % 8 || sg.tap_stride % 8) return false;
    if (reinterpret_cast<uintptr_t>(sg.base) & 15) return false;
  }
  const int hpt = epi == EPI_GLOBAL ? (p.heads < 4 ? p.heads : 4) : 1;
  return tch_smem_bytes(epi, p.J, p.fpt, hpt) <= TC_SMEM_MAX;
}

inline int tc_launch_h(cudaStream_t st, int epi, const GemmP& p, const TcWeights& t) {
  if (!t.f16 || epi == EPI_GLOBAL) return -1;
  const dim3 grid((unsigned)(((p.F + p.fpt - 1) / p.fpt) * ((p.N + TC_BN - 1) / TC_BN)));
  const int hpt = epi == EPI_GLOBAL ? (p.heads < 4 ? p.heads : 4) : 1;
  const size_t smem = tch_smem_bytes(epi, p.J, p.fpt, hpt);
  const auto kernel = epi == EPI_PLAIN ? gemm_tc_h_kernel<EPI_PLAIN> : gemm_tc_h_kernel<EPI_SEMCH>;
  static bool attr_set[64][3];
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63][epi]) {
    cudaError_t e = cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev & 63][epi] = true;
  }
  TcActMaps am{};
  const long long rows = (long long)p.F * p.J;
  for (int s = 0; s < p.nseg; ++s)
    if (tc_seg_tma_h(p.seg[s]) && tc_encode_a16(&am.seg[s], p.seg[s].base, p.seg[s].Kc, rows, p.seg[s].ld)) return -1;
  if (epi == EPI_PLAIN && tc_encode_rows16(&am.out, p.out, p.N, rows, p.ld_out, p.fpt * p.J)) return -1;
  kernel<<<grid, TC_THREADS, smem, st>>>(p, t.map_h16hi, am, t.sw);
  return (int)cudaGetLastError();
}

template <int PREC>
inline int tc_launch_prec(cudaStream_t st, int epi, const GemmP& p, const TcWeights& t) {
  const int tiles = ((p.F + p.fpt - 1) / p.fpt) * ((p.N + TC_BN - 1) / TC_BN);
  const int hpt = epi == EPI_GLOBAL ? (p.heads < 4 ? p.heads : 4) : 1;
  const size_t smem = tc_smem_bytes(PREC, epi, p.J, p.fpt, hpt);
  const auto kernel = with_epi(epi, [](auto e) { return gemm_tc_kernel<decltype(e)::value, PREC>; });
  static bool attr_set[64][3];              // the shared-memory opt-in is per device
  static int sms[64];
  int dev = 0;
  cudaGetDevice(&dev);
  if (!attr_set[dev & 63][epi]) {
    cudaError_t e = cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_OPTIN);
    if (e != cudaSuccess) return (int)e;
    e = cudaDeviceGetAttribute(&sms[dev & 63], cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev & 63][epi] = true;
  }
  // the persistent form takes one CTA per SM at most, the others one per tile
  const dim3 grid((unsigned)(tc_persistent(epi) && tiles > sms[dev & 63] ? sms[dev & 63] : tiles));
  const CUtensorMap& mhi = PREC == TC_F16X3 ? t.map_h16hi : t.map_hi;
  const CUtensorMap& mlo = PREC == TC_F16X3 ? t.map_h16lo : t.map_lo;
  // the activation maps follow the pointers, so they are encoded per launch (graph capture keeps them by value)
  TcActMaps am{};
  const long long rows = (long long)p.F * p.J;
  for (int s = 0; s < p.nseg; ++s)
    if (tc_seg_tma(p.seg[s]) && tc_encode_taps(&am.seg[s], p.seg[s], p.F, p.J, p.fpt)) return -1;
  if (epi == EPI_PLAIN && tc_encode_rows(&am.out, p.out, p.N, rows, p.ld_out, p.fpt * p.J)) return -1;
  CUtensorMap mres{};
  if (epi == EPI_PLAIN && tc_res_tma(p)) {
    ASeg r;                                  // the residual as a one-tap segment of N columns at its frame map
    r.base = p.res; r.ld = p.res_ld; r.K = r.Kc = p.N; r.tap_stride = 0; r.map = p.res_map;
    if (tc_encode_taps(&mres, r, p.F, p.J, p.fpt)) return -1;
  }
  if (epi == EPI_SEMCH && tc_encode_semch(&am.out, p.out, p.C, p.N / (TC_BN * p.tiles_per_mask), rows, p.ld_out,
                                          p.fpt * p.J))
    return -1;
  kernel<<<grid, TC_THREADS, smem, st>>>(p, mhi, mlo, am, t.sw, mres);
  return (int)cudaGetLastError();
}

// Tiles in the order tile = row tile * column tiles + column tile (the column tile fastest, see gemm_tc_kernel).
// prec: TC_3XTF32 (needs t.f16 false), TC_1XTF32, TC_F16X3 or TC_F16 (both need t.f16).
inline int tc_launch(cudaStream_t st, int epi, const GemmP& p, const TcWeights& t, int prec) {
  if (prec == TC_F16) return tc_launch_h(st, epi, p, t);
  if (prec == TC_1XTF32) return tc_launch_prec<TC_1XTF32>(st, epi, p, t);
  if (prec == TC_F16X3) return t.f16 ? tc_launch_prec<TC_F16X3>(st, epi, p, t) : -1;
  return t.f16 ? -1 : tc_launch_prec<TC_3XTF32>(st, epi, p, t);
}

// The fp32-grade form of a weight copy: F16X3 for inference's copies, 3xTF32 for training's
inline int tc_prec(const TcWeights& t, int precision) {
  return precision == 1 ? TC_1XTF32 : t.f16 ? TC_F16X3 : TC_3XTF32;
}

}  // namespace gast
