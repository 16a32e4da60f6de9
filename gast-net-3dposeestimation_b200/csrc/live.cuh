// The live tick's own steps (gen_img_kpts, lib/pose/hrnet/pose_estimation/gen_kpts.py:115-175, feeding the causal
// real-time models of gen_skes.py:43-69, placed by revise_skes_real_time, tools/preprocess.py:158-172) for C cameras
// of num_person slots each (DESIGN.md §8.10):
//   gast_live_slots   gast_sort_update's rows of one frame per camera -> the selected tracks bound to slots by id, and
//                     each active slot's crop geometry: center and scale, the forward and the inverse matrix;
//   gast_live_inputs  the decoded COCO keypoints of every slot -> H36M keypoints and scores, the limb repair, the
//                     stream pool's normalised input row and its device fresh and active masks;
//   gast_live_place   the lifted world poses -> each camera's active persons placed, the height rebased over them.
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
