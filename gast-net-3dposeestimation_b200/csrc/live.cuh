// The live tick's own steps (gen_img_kpts, lib/pose/hrnet/pose_estimation/gen_kpts.py:115-175, feeding the causal
// real-time models of gen_skes.py:43-69, placed by revise_skes_real_time, tools/preprocess.py:158-172) for C cameras
// of num_person slots each (DESIGN.md §8.10):
//   gast_live_slots   gast_sort_update's rows of one frame per camera -> the selected tracks bound to slots by id, and
//                     each active slot's crop geometry: center and scale, the forward and the inverse matrix;
//   gast_live_inputs  the decoded COCO keypoints of every slot -> H36M keypoints and scores, the limb repair, the
//                     stream pool's normalised input row and its device fresh and active masks;
//   gast_live_place   the lifted world poses -> each camera's active persons placed, the height rebased over them.
// and, for the non-causal models' delayed tick (DESIGN.md §8.11):
//   gast_live_delayed_inputs  gast_live_inputs plus each slot's sequence: its id, last push, length, the gap rule and
//                             the tail mask of the sequences that end this tick;
//   gast_live_delayed_end     the tail mask of every pending sequence of the listed cameras (end());
//   gast_live_delayed_place   the final, provisional and tail poses placed with the keypoints of their own frames,
//                             from a per-slot ring of repaired keypoints and frame ticks.
// The formulas are box_geometry.cuh's and pipeline.cuh's own device functions; nothing is restated here.  No atomics
// and no allocation: every value has one writer, so ticks repeat bit for bit and can be captured in a CUDA graph.
//
// Included at the end of gast_api.cu (uses fail / CUDA_OK / cdiv, box_geometry.cuh, pipeline.cuh).
#pragma once
#include "box_geometry.cuh"

namespace gast {

constexpr int LIVE_MAX_PERSON = 32;       // one lane per slot in gast_live_slots
constexpr int LIVE_STATUS_WORDS = 16;     // per camera: word, ticks, first tick of status bits 0 .. 11, 2 spare
constexpr int LIVE_STATUS_BITS = 12;
constexpr int LIVE_INPUT_WARPS = 4;
constexpr int LIVE_PLACE_THREADS = 256;

// One warp per camera.  Lane 0 keeps the slot book: the selected ids (gen_img_kpts:146-150, no round(v, 2)) that hold
// a slot keep it; the others take, in selection order, the free slots in ascending order, then the slots not selected
// this tick with the oldest last-seen tick (lowest slot first).  A slot whose id changes needs a fresh stream.  Lane p
// then computes slot p's geometry.  book (3, C, P) int64: id (-1 none), last tick seen (-1 never), needs fresh.
__global__ void __launch_bounds__(32)
live_slots_kernel(const double* __restrict__ rows, const int* __restrict__ counts, const int* __restrict__ sort_status,
                  int cap, int P, int W, int H, int ow, int oh, int hw, int hh, long long* __restrict__ book,
                  long long* __restrict__ status, int* __restrict__ slot_active, double* __restrict__ fwd_out,
                  double* __restrict__ inv_out, float* __restrict__ cs_out) {
  __shared__ int sh_row[LIVE_MAX_PERSON], slot_of[LIVE_MAX_PERSON];
  const int c = blockIdx.x, lane = threadIdx.x, C = gridDim.x;
  long long* st = status + (long long)c * LIVE_STATUS_WORDS;
  const long long tick = st[1];
  const int k = counts[c];
  const int n = rec_count(k, P, cap);
  long long* ids = book + (long long)c * P;
  long long* seen = ids + (long long)C * P;
  long long* fresh = seen + (long long)C * P;
  const double* fr = rows + (long long)c * cap * 5;
  if (lane == 0) {
    unsigned taken = 0;
    for (int i = 0; i < n; ++i) {
      const long long id = (long long)fr[(k == 1 ? 0 : k - 1 - i) * 5 + 4];
      slot_of[i] = -1;
      for (int s = 0; s < P; ++s)
        if (ids[s] == id && !(taken >> s & 1u)) {
          slot_of[i] = s;
          taken |= 1u << s;
          break;
        }
    }
    for (int i = 0; i < n; ++i) {
      if (slot_of[i] >= 0) continue;
      int pick = -1;
      for (int s = 0; s < P && pick < 0; ++s)
        if (ids[s] < 0 && !(taken >> s & 1u)) pick = s;
      for (int s = 0; s < P && pick < 0; ++s) {   // there is room: at most P ids are selected
        if (taken >> s & 1u) continue;
        bool oldest = true;
        for (int q = 0; q < P; ++q)
          if (!(taken >> q & 1u) && seen[q] < seen[s]) oldest = false;
        if (oldest) pick = s;
      }
      slot_of[i] = pick;
      taken |= 1u << pick;
      ids[pick] = (long long)fr[(k == 1 ? 0 : k - 1 - i) * 5 + 4];
      fresh[pick] = 1;
    }
    for (int s = 0; s < P; ++s) sh_row[s] = -1;
    for (int i = 0; i < n; ++i) {
      sh_row[slot_of[i]] = k == 1 ? 0 : k - 1 - i;
      seen[slot_of[i]] = tick;
    }
  }
  __syncwarp();
  int bits = 0;
  if (lane < P) {
    const int r = sh_row[lane];
    const long long o = (long long)c * P + lane;
    double m[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, mi[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    float c0 = 0.f, c1 = 0.f, s0 = 0.f, s1 = 0.f;
    bool active = false;
    if (r >= 0) {
      const double* row = fr + r * 5;
      int box_bits = 0;
      rec_center_scale(row[0], row[1], row[2], row[3], __ddiv_rn((double)H, (double)W), box_bits, c0, c1, s0, s1);
      float src[6], dst[6];
      rec_triangles(c0, c1, s0, ow, oh, src, dst);
      rec_affine(src, dst, m);
      bool finite = true;
#pragma unroll
      for (int i = 0; i < 6; ++i) finite &= isfinite(m[i]);
      if (!finite) box_bits |= REC_ST_MATRIX;
      active = box_bits == 0;
      bits = box_bits;
      if (active && hw > 0) {
        float dh[6];
        rec_triangles(c0, c1, s0, hw, hh, src, dh);
        rec_affine(dh, src, mi);
      }
      if (!active) {
        c0 = c1 = s0 = s1 = 0.f;
#pragma unroll
        for (int i = 0; i < 6; ++i) m[i] = 0.0;
      }
    }
#pragma unroll
    for (int i = 0; i < 6; ++i) fwd_out[6 * o + i] = m[i];
    if (hw > 0)
#pragma unroll
      for (int i = 0; i < 6; ++i) inv_out[6 * o + i] = mi[i];
    reinterpret_cast<float4*>(cs_out)[o] = make_float4(c0, c1, s0, s1);
    slot_active[o] = active ? 1 : 0;
  }
#pragma unroll
  for (int q = 16; q > 0; q >>= 1) bits |= __shfl_xor_sync(0xffffffffu, bits, q);
  if (lane == 0) {
    bits |= (n < 0 ? REC_ST_TRACKS : 0) | sort_status[c];
    const long long word = st[0];
    for (int b = 0; b < LIVE_STATUS_BITS; ++b)
      if ((bits >> b & 1) && !(word >> b & 1)) st[2 + b] = tick;
    st[0] = word | bits;
    st[1] = tick + 1;
  }
}

// One warp per slot.  Lane 0 converts the slot's decoded keypoints and scores (h36m_coco_format), tests keep and
// valid, and repairs the limbs (revise_kpts); the lanes write the keypoints, the scores and the normalised input row.
// A slot is active when its box was, keep and valid hold; an inactive slot's rows are zero.  The masks are the stream
// pool's, for both library halves with test-time augmentation (copies = 2: stream s and its twin s + N).
__global__ void __launch_bounds__(LIVE_INPUT_WARPS * 32)
live_inputs_kernel(const float* __restrict__ preds, const float* __restrict__ maxvals, const int* __restrict__ slot_active,
                   int N, float w, double hw, int copies, long long* __restrict__ fresh_book, float* __restrict__ kpts_out,
                   float* __restrict__ scores_out, float* __restrict__ x_out, int* __restrict__ fresh_mask,
                   int* __restrict__ active_mask, unsigned char* __restrict__ active_out) {
  __shared__ float sh_k[LIVE_INPUT_WARPS][34], sh_s[LIVE_INPUT_WARPS][17];
  __shared__ int sh_act[LIVE_INPUT_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s = blockIdx.x * LIVE_INPUT_WARPS + warp;
  if (s >= N) return;
  if (lane == 0) {
    const float* k = preds + (long long)s * 34;
    float h[34], n[17];
    coco_to_h36m_frame(k, 2, h);
    coco_scores_to_h36m(maxvals + (long long)s * 17, n);
    const bool act = slot_active[s] && coco_any_nonzero(k) && np_pairwise_sum(h, 34) != 0.f;
    revise_kpts_frame(reinterpret_cast<const float2*>(h), n, reinterpret_cast<float2*>(sh_k[warp]), 17);
#pragma unroll
    for (int j = 0; j < 17; ++j) sh_s[warp][j] = n[j];
    sh_act[warp] = act;
    const int need = (int)fresh_book[s];
    for (int q = 0; q < copies; ++q) {
      fresh_mask[s + q * N] = act && need;
      active_mask[s + q * N] = act;
    }
    if (act) fresh_book[s] = 0;
    active_out[s] = act;
  }
  __syncwarp();
  const bool act = sh_act[warp];
  for (int i = lane; i < 34; i += 32) {
    const float v = act ? sh_k[warp][i] : 0.f;
    kpts_out[(long long)s * 34 + i] = v;
    x_out[(long long)s * 34 + i] = act ? screen_norm(v, w, (i & 1) ? hw : 1.0) : 0.f;
  }
  if (lane < 17) scores_out[(long long)s * 17 + lane] = act ? sh_s[warp][lane] : 0.f;
}

// One CTA per camera: revise_skes_real_time over the camera's active slots in slot order, z -= the NaN-propagating
// minimum of their z; inactive slots are zero.
__global__ void __launch_bounds__(LIVE_PLACE_THREADS)
live_place_kernel(const float* __restrict__ world, const float* __restrict__ kpts, const unsigned char* __restrict__ active,
                  int P, float cx, float cy, float r, float* __restrict__ out) {
  __shared__ float sh[LIVE_PLACE_THREADS / 32];
  const int c = blockIdx.x, tid = threadIdx.x;
  const long long base = (long long)c * P;
  float z = INFINITY;
  for (int i = tid; i < P * 17; i += LIVE_PLACE_THREADS)
    if (active[base + i / 17]) z = np_minf(world[(base * 17 + i) * 3 + 2], z);
  for (int o = 16; o > 0; o >>= 1) z = np_minf(__shfl_xor_sync(0xffffffffu, z, o), z);
  if ((tid & 31) == 0) sh[tid >> 5] = z;
  __syncthreads();
  float zmin = sh[0];
  for (int q = 1; q < LIVE_PLACE_THREADS / 32; ++q) zmin = np_minf(sh[q], zmin);
  for (int i = tid; i < P * 17; i += LIVE_PLACE_THREADS) {
    const long long p = base + i / 17, e = base * 17 + i;
    float x = 0.f, y = 0.f, zz = 0.f;
    if (active[p]) {
      rt_place(world + 3 * e, kpts + p * 34, 2, cx, cy, r, x, y);
      zz = __fsub_rn(world[3 * e + 2], zmin);
    }
    out[3 * e] = x;
    out[3 * e + 1] = y;
    out[3 * e + 2] = zz;
  }
}

// ---- the delayed tick of the non-causal models (DESIGN.md §8.11) ------------------------------------------------------
// seq (4, n) int64 per slot: the SORT id of its stream's current sequence (-1 none), the tick of its last push (-1
// never), the frames of that sequence (0: none pending) and the length of the sequence that ended this tick (0: none).

// live_inputs_kernel's conversion, repair and masks, and each slot's sequence: a slot ends its sequence when it pushes
// with the restart flag set (a new id took it) or, with max_gap >= 0, when it has not pushed for more than max_gap ticks;
// either way only with frames pending.  The tail mask marks the ending streams (both halves with copies = 2).  A gap end
// sets the restart flag, so the id's next push starts a new sequence.
__global__ void __launch_bounds__(LIVE_INPUT_WARPS * 32)
live_delayed_inputs_kernel(const float* __restrict__ preds, const float* __restrict__ maxvals,
                           const int* __restrict__ slot_active, int N, int P, float w, double hw, int copies,
                           long long max_gap, const long long* __restrict__ status, long long* __restrict__ book,
                           long long* __restrict__ seq, float* __restrict__ kpts_out, float* __restrict__ scores_out,
                           float* __restrict__ x_out, int* __restrict__ fresh_mask, int* __restrict__ active_mask,
                           int* __restrict__ tail_mask, unsigned char* __restrict__ active_out,
                           long long* __restrict__ tail_ids) {
  __shared__ float sh_k[LIVE_INPUT_WARPS][34], sh_s[LIVE_INPUT_WARPS][17];
  __shared__ int sh_act[LIVE_INPUT_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int s = blockIdx.x * LIVE_INPUT_WARPS + warp;
  if (s >= N) return;
  if (lane == 0) {
    const float* k = preds + (long long)s * 34;
    float h[34], n[17];
    coco_to_h36m_frame(k, 2, h);
    coco_scores_to_h36m(maxvals + (long long)s * 17, n);
    const bool act = slot_active[s] && coco_any_nonzero(k) && np_pairwise_sum(h, 34) != 0.f;
    revise_kpts_frame(reinterpret_cast<const float2*>(h), n, reinterpret_cast<float2*>(sh_k[warp]), 17);
#pragma unroll
    for (int j = 0; j < 17; ++j) sh_s[warp][j] = n[j];
    sh_act[warp] = act;
    long long* fresh_book = book + 2LL * N;
    long long *id = seq + s, *last = id + N, *len = last + N, *tail_len = len + N;
    const long long tick = status[(long long)(s / P) * LIVE_STATUS_WORDS + 1] - 1;   // gast_live_slots counted it
    const bool need = fresh_book[s] != 0;
    const long long pending = *len;
    const bool gap = !act && pending >= 1 && max_gap >= 0 && tick - *last > max_gap;
    const bool ending = pending >= 1 && (gap || (act && need));
    for (int q = 0; q < copies; ++q) {
      fresh_mask[s + q * N] = act && need;
      active_mask[s + q * N] = act;
      tail_mask[s + q * N] = ending;
    }
    *tail_len = ending ? pending : 0;
    tail_ids[s] = ending ? *id : -1;
    if (act) {
      if (need) *id = book[s];
      *len = (need ? 0 : pending) + 1;
      *last = tick;
      fresh_book[s] = 0;
    }
    if (gap) {
      *len = 0;
      fresh_book[s] = 1;
    }
    active_out[s] = act;
  }
  __syncwarp();
  const bool act = sh_act[warp];
  for (int i = lane; i < 34; i += 32) {
    const float v = act ? sh_k[warp][i] : 0.f;
    kpts_out[(long long)s * 34 + i] = v;
    x_out[(long long)s * 34 + i] = act ? screen_norm(v, w, (i & 1) ? hw : 1.0) : 0.f;
  }
  if (lane < 17) scores_out[(long long)s * 17 + lane] = act ? sh_s[warp][lane] : 0.f;
}

// end(cameras): every slot of a listed camera (cameras (C) uint8) with frames pending ends its sequence
__global__ void live_delayed_end_kernel(const unsigned char* __restrict__ cameras, int N, int P, int copies,
                                        long long* __restrict__ seq, int* __restrict__ tail_mask,
                                        long long* __restrict__ tail_ids) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= N) return;
  const long long pending = seq[2LL * N + s];
  const bool ending = cameras[s / P] && pending >= 1;
  for (int q = 0; q < copies; ++q) tail_mask[s + q * N] = ending;
  seq[3LL * N + s] = ending ? pending : 0;
  tail_ids[s] = ending ? seq[s] : -1;
}

// the NaN-propagating minimum of every thread's z over the CTA (every thread calls it; sh holds one float per warp)
__device__ __forceinline__ float live_cta_zmin(float z, float* sh) {
  for (int o = 16; o > 0; o >>= 1) z = np_minf(__shfl_xor_sync(0xffffffffu, z, o), z);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = z;
  __syncthreads();
  float zmin = sh[0];
  for (int q = 1; q < LIVE_PLACE_THREADS / 32; ++q) zmin = np_minf(sh[q], zmin);
  __syncthreads();
  return zmin;
}

// One group of a camera's slots placed together (revise_skes_real_time, z rebased over the group): slot p of the camera
// belongs to it when it pushed this tick and its frame at position len - 1 - behind exists; its pose is row `row` of the
// rows_per_slot world rows of the slot, placed with that frame's keypoints (the ring's, or this tick's for the newest).
__device__ __forceinline__ void live_place_group(const float* __restrict__ world, int rows_per_slot, int behind,
                                                 const float* __restrict__ kpts, const unsigned char* __restrict__ active,
                                                 const long long* __restrict__ len, const float* __restrict__ ring_kpts,
                                                 const long long* __restrict__ ring_ticks, int R, long long base, int P,
                                                 long long tick, float cx, float cy, float r, float* __restrict__ out,
                                                 long long* __restrict__ frame, float* sh) {
  const int tid = threadIdx.x;
  float z = INFINITY;
  for (int i = tid; i < P * 17; i += LIVE_PLACE_THREADS) {
    const long long p = base + i / 17;
    if (active[p] && len[p] - 1 - behind >= 0)
      z = np_minf(world[((p * rows_per_slot + rows_per_slot - 1) * 17 + i % 17) * 3 + 2], z);
  }
  const float zmin = live_cta_zmin(z, sh);
  for (int i = tid; i < P * 17; i += LIVE_PLACE_THREADS) {
    const long long p = base + i / 17, e = base * 17 + i;
    const long long pos = active[p] ? len[p] - 1 - behind : -1;
    float x = 0.f, y = 0.f, zz = 0.f;
    long long f = -1;
    if (pos >= 0) {
      const long long slot = p * R + pos % R;
      const bool newest = pos == len[p] - 1;
      const float* w = world + ((p * rows_per_slot + rows_per_slot - 1) * 17 + i % 17) * 3;
      rt_place(w, newest ? kpts + p * 34 : ring_kpts + slot * 34, 2, cx, cy, r, x, y);
      zz = __fsub_rn(w[2], zmin);
      f = newest ? tick : ring_ticks[slot];
    }
    out[3 * e] = x;
    out[3 * e + 1] = y;
    out[3 * e + 2] = zz;
    if (i % 17 == 0) frame[p] = f;
  }
}

// One CTA per camera: the final poses (latency pushes behind), the provisional poses (lookahead >= 0: that many
// behind), then each ended sequence's tail rows placed one by one, and last the ring written with this tick's frames
// (after every read of the ring: a restarting slot's first frame lands where its old sequence's tail may be).  active
// null: no slot pushed (end), so only the tails are written.
__global__ void __launch_bounds__(LIVE_PLACE_THREADS)
live_delayed_place_kernel(const float* __restrict__ world, const float* __restrict__ world_tail,
                          const float* __restrict__ world_now, int now_rows, const float* __restrict__ kpts,
                          const unsigned char* __restrict__ active, const long long* __restrict__ seq,
                          const long long* __restrict__ status, int P, int latency, int lookahead, float cx, float cy,
                          float r, float* __restrict__ ring_kpts, long long* __restrict__ ring_ticks,
                          float* __restrict__ poses, long long* __restrict__ frame, float* __restrict__ now,
                          long long* __restrict__ now_frame, float* __restrict__ tail, long long* __restrict__ tail_frame) {
  __shared__ float sh[LIVE_PLACE_THREADS / 32];
  const int c = blockIdx.x, tid = threadIdx.x, R = latency + 1;
  const long long N = (long long)gridDim.x * P, base = (long long)c * P;
  const long long* len = seq + 2 * N;
  const long long* tail_len = seq + 3 * N;
  const long long tick = status[(long long)c * LIVE_STATUS_WORDS + 1] - 1;
  if (active) {
    live_place_group(world, 1, latency, kpts, active, len, ring_kpts, ring_ticks, R, base, P, tick, cx, cy, r, poses,
                     frame, sh);
    if (lookahead >= 0)
      live_place_group(world_now, now_rows, lookahead, kpts, active, len, ring_kpts, ring_ticks, R, base, P, tick, cx,
                       cy, r, now, now_frame, sh);
  }
  for (int i = tid; i < P * latency; i += LIVE_PLACE_THREADS) {
    const long long p = base + i / latency, row = base * latency + i;
    const long long pos = tail_len[p] - latency + i % latency;   // tail_len 0: no tail, every pos < 0
    const float* wr = world_tail + row * 51;
    float* o = tail + row * 51;
    if (pos >= 0) {
      const long long slot = p * R + pos % R;
      float zmin = INFINITY;
      for (int j = 0; j < 17; ++j) zmin = np_minf(wr[3 * j + 2], zmin);
      for (int j = 0; j < 17; ++j) {
        float x, y;
        rt_place(wr + 3 * j, ring_kpts + slot * 34, 2, cx, cy, r, x, y);
        o[3 * j] = x;
        o[3 * j + 1] = y;
        o[3 * j + 2] = __fsub_rn(wr[3 * j + 2], zmin);
      }
      tail_frame[row] = ring_ticks[slot];
    } else {
      for (int j = 0; j < 51; ++j) o[j] = 0.f;
      tail_frame[row] = -1;
    }
  }
  if (!active) return;
  __syncthreads();
  for (int i = tid; i < P * 34; i += LIVE_PLACE_THREADS) {
    const long long p = base + i / 34;
    if (!active[p]) continue;
    const long long slot = p * R + (len[p] - 1) % R;
    ring_kpts[slot * 34 + i % 34] = kpts[p * 34 + i % 34];
    if (i % 34 == 0) ring_ticks[slot] = tick;
  }
}

}  // namespace gast

extern "C" int gast_live_slots(const double* rows, const int32_t* counts, const int32_t* sort_status, int32_t C,
                               int32_t capacity, int32_t num_person, int32_t W, int32_t H, int32_t out_w,
                               int32_t out_h, int32_t hw, int32_t hh, int64_t* book, int64_t* status,
                               int32_t* slot_active, double* forward_mats, double* inverse_mats, float* center_scale,
                               void* stream) {
  using namespace gast;
  if (!rows || !counts || !sort_status || !book || !status || !slot_active || !forward_mats || !center_scale || C < 1 ||
      capacity < 1 || num_person < 1 || num_person > LIVE_MAX_PERSON)
    return fail("gast_live_slots: bad arguments (1 <= num_person <= %d)", LIVE_MAX_PERSON);
  if (W < 1 || H < 1 || W > REC_MAX_SIDE || H > REC_MAX_SIDE || out_w < 1 || out_h < 1 || out_w > REC_MAX_SIDE ||
      out_h > REC_MAX_SIDE)
    return fail("gast_live_slots: a %d x %d frame or a %d x %d crop (each side 1 .. %d)", W, H, out_w, out_h,
                REC_MAX_SIDE);
  if (!((hw == 0 && hh == 0) || (hw >= 1 && hh >= 1 && hw <= REC_MAX_SIDE && hh <= REC_MAX_SIDE && inverse_mats)))
    return fail("gast_live_slots: a %d x %d heatmap (0 x 0, or each side 1 .. %d with inverse_mats)", hw, hh,
                REC_MAX_SIDE);
  live_slots_kernel<<<C, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      rows, counts, sort_status, capacity, num_person, W, H, out_w, out_h, hw, hh, reinterpret_cast<long long*>(book),
      reinterpret_cast<long long*>(status), slot_active, forward_mats, inverse_mats, center_scale);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_live_inputs(const float* preds, const float* maxvals, const int32_t* slot_active, int32_t n,
                                int32_t W, int32_t H, int32_t copies, int64_t* book_fresh, float* kpts, float* scores,
                                float* x, int32_t* fresh_mask, int32_t* active_mask, uint8_t* active, void* stream) {
  using namespace gast;
  if (!preds || !maxvals || !slot_active || !book_fresh || !kpts || !scores || !x || !fresh_mask || !active_mask ||
      !active || n < 1 || W < 1 || H < 1 || (copies != 1 && copies != 2))
    return fail("gast_live_inputs: bad arguments");
  live_inputs_kernel<<<cdiv(n, LIVE_INPUT_WARPS), LIVE_INPUT_WARPS * 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      preds, maxvals, slot_active, n, (float)W, (double)(float)H / (double)(float)W, copies,
      reinterpret_cast<long long*>(book_fresh), kpts, scores, x, fresh_mask, active_mask, active);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_live_place(const float* world, const float* kpts, const uint8_t* active, int32_t C,
                               int32_t num_person, double width, float* out, void* stream) {
  using namespace gast;
  if (!world || !kpts || !active || !out || C < 1 || num_person < 1 || !(width > 0.0))
    return fail("gast_live_place: bad arguments");
  float cx, cy, r;
  rt_constants(width, cx, cy, r);
  live_place_kernel<<<C, LIVE_PLACE_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(world, kpts, active,
                                                                                         num_person, cx, cy, r, out);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_live_delayed_inputs(const float* preds, const float* maxvals, const int32_t* slot_active, int32_t C,
                                        int32_t num_person, int32_t W, int32_t H, int32_t copies, int32_t max_gap,
                                        const int64_t* status, int64_t* book, int64_t* seq, float* kpts, float* scores,
                                        float* x, int32_t* fresh_mask, int32_t* active_mask, int32_t* tail_mask,
                                        uint8_t* active, int64_t* tail_ids, void* stream) {
  using namespace gast;
  if (!preds || !maxvals || !slot_active || !status || !book || !seq || !kpts || !scores || !x || !fresh_mask ||
      !active_mask || !tail_mask || !active || !tail_ids || C < 1 || num_person < 1 || num_person > LIVE_MAX_PERSON ||
      W < 1 || H < 1 || (copies != 1 && copies != 2) || max_gap < -1)
    return fail("gast_live_delayed_inputs: bad arguments (1 <= num_person <= %d, max_gap >= -1)", LIVE_MAX_PERSON);
  const int n = C * num_person;
  live_delayed_inputs_kernel<<<cdiv(n, LIVE_INPUT_WARPS), LIVE_INPUT_WARPS * 32, 0,
                               reinterpret_cast<cudaStream_t>(stream)>>>(
      preds, maxvals, slot_active, n, num_person, (float)W, (double)(float)H / (double)(float)W, copies, max_gap,
      reinterpret_cast<const long long*>(status), reinterpret_cast<long long*>(book), reinterpret_cast<long long*>(seq),
      kpts, scores, x, fresh_mask, active_mask, tail_mask, active, reinterpret_cast<long long*>(tail_ids));
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_live_delayed_end(const uint8_t* cameras, int32_t C, int32_t num_person, int32_t copies,
                                     int64_t* seq, int32_t* tail_mask, int64_t* tail_ids, void* stream) {
  using namespace gast;
  if (!cameras || !seq || !tail_mask || !tail_ids || C < 1 || num_person < 1 || num_person > LIVE_MAX_PERSON ||
      (copies != 1 && copies != 2))
    return fail("gast_live_delayed_end: bad arguments");
  const int n = C * num_person;
  live_delayed_end_kernel<<<cdiv(n, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      cameras, n, num_person, copies, reinterpret_cast<long long*>(seq), tail_mask,
      reinterpret_cast<long long*>(tail_ids));
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_live_delayed_place(const float* world, const float* world_tail, const float* world_now,
                                       int32_t now_rows, const float* kpts, const uint8_t* active, const int64_t* seq,
                                       const int64_t* status, int32_t C, int32_t num_person, int32_t latency,
                                       int32_t lookahead, double width, float* ring_kpts, int64_t* ring_ticks,
                                       float* poses, int64_t* frame, float* now, int64_t* now_frame, float* tail,
                                       int64_t* tail_frame, void* stream) {
  using namespace gast;
  if (!world_tail || !seq || !status || !ring_kpts || !ring_ticks || !tail || !tail_frame || C < 1 || num_person < 1 ||
      latency < 1 || !(width > 0.0))
    return fail("gast_live_delayed_place: bad arguments");
  if (active && (!world || !kpts || !poses || !frame || lookahead < -1 || lookahead >= latency ||
                 (lookahead >= 0 && (!world_now || !now || !now_frame || now_rows != latency - lookahead))))
    return fail("gast_live_delayed_place: bad final or provisional arguments (lookahead %d, %d rows, latency %d)",
                lookahead, now_rows, latency);
  float cx, cy, r;
  rt_constants(width, cx, cy, r);
  live_delayed_place_kernel<<<C, LIVE_PLACE_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      world, world_tail, world_now, now_rows, kpts, active, reinterpret_cast<const long long*>(seq),
      reinterpret_cast<const long long*>(status), num_person, latency, active ? lookahead : -1, cx, cy, r, ring_kpts,
      reinterpret_cast<long long*>(ring_ticks), poses, reinterpret_cast<long long*>(frame), now,
      reinterpret_cast<long long*>(now_frame), tail, reinterpret_cast<long long*>(tail_frame));
  CUDA_OK(cudaGetLastError());
  return 0;
}
