// SORT's tracks to the 2D pose net's crop records (lib/pose/hrnet/pose_estimation/gen_kpts.py:214-256): the boxes
// gen_video_kpts keeps of each frame, their round(v, 2), box_to_center_scale and get_affine_transform, on the device.
//   gast_track_records  gast_sort_update's rows of S sequences x K frames -> one record per kept box: its frame, its
//                       output slot, the forward (frame -> crop) matrix, and its center and scale;
//   gast_record_inverse the records' inverse (heatmap -> frame) matrices for a heatmap size.
//
// The geometry itself is box_geometry.cuh's, shared with the live tick (live.cuh).
//
// gast_track_records runs one CTA per sequence.  The CTA first sums the record counts of the sequences before it
// (S * K integer reads), so the records of all sequences are contiguous without a second launch or scratch; then it
// walks its frames in tiles of the block, one thread per frame, with block scans for the record offsets and the kept
// frames' ranks.  No atomics: calls repeat bit for bit, and a sequence's records do not depend on the other
// sequences' rows.
//
// Included at the end of gast_api.cu (uses fail / CUDA_OK / cdiv).
#pragma once
#include "box_geometry.cuh"

namespace gast {

constexpr int REC_THREADS = 256;
constexpr int REC_WARPS = REC_THREADS / 32;
constexpr int REC_INV_THREADS = 128;
constexpr int REC_MAX_SIDE = 32767;

// inclusive block scan of two counters; returns the block totals
__device__ __forceinline__ int2 rec_block_scan(int2& v, int2* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int x = __shfl_up_sync(0xffffffffu, v.x, o), y = __shfl_up_sync(0xffffffffu, v.y, o);
    if (lane >= o) {
      v.x += x;
      v.y += y;
    }
  }
  if (lane == 31) sh[warp] = v;
  __syncthreads();
  int2 before = make_int2(0, 0), total = make_int2(0, 0);
#pragma unroll
  for (int w = 0; w < REC_WARPS; ++w) {
    if (w < warp) {
      before.x += sh[w].x;
      before.y += sh[w].y;
    }
    total.x += sh[w].x;
    total.y += sh[w].y;
  }
  __syncthreads();
  v.x += before.x;
  v.y += before.y;
  return total;
}

__global__ void __launch_bounds__(REC_THREADS, 1)
track_records_kernel(const double* __restrict__ rows, const int* __restrict__ counts, const int* __restrict__ status,
                     int K, int cap, int num_person, int W, int H, int ow, int oh, int S, int* __restrict__ frame_out,
                     long long* __restrict__ slot_out, double* __restrict__ fwd_out, float* __restrict__ cs_out,
                     int* __restrict__ summary, int* __restrict__ total_out) {
  __shared__ int2 sh_scan[REC_WARPS];
  __shared__ int sh_red[REC_WARPS][3];
  const int s = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // the records of the sequences before this one
  int before = 0;
  for (long long f = tid; f < (long long)s * K; f += REC_THREADS) before += max(rec_count(counts[f], num_person, cap), 0);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) before += __shfl_xor_sync(0xffffffffu, before, o);
  if (lane == 0) sh_red[warp][0] = before;
  __syncthreads();
  long long base = 0;
#pragma unroll
  for (int w = 0; w < REC_WARPS; ++w) base += sh_red[w][0];
  __syncthreads();

  // box_to_center_scale with (H, W) in the model-size slots, as PreProcess calls it
  const double aspect = __ddiv_rn((double)H, (double)W);
  long long rec_done = 0;
  int kept_done = 0, bits = 0, first = K;
  for (int t0 = 0; t0 < K; t0 += REC_THREADS) {
    const int t = t0 + tid;
    const long long fr = (long long)s * K + t;
    const int k = t < K ? counts[fr] : 0;
    const int n = t < K ? rec_count(k, num_person, cap) : 0;
    int my_bits = n < 0 ? REC_ST_TRACKS : 0;
    int2 v = make_int2(max(n, 0), n > 0 ? 1 : 0);
    const int2 tile = rec_block_scan(v, sh_scan);
    const long long at = base + rec_done + v.x - max(n, 0);
    const int rank = kept_done + v.y - (n > 0 ? 1 : 0);
    for (int p = 0; p < n; ++p) {
      const double* row = rows + (fr * cap + (k == 1 ? 0 : k - 1 - p)) * 5;
      // np.round(v, 2): rint(v * 100) / 100
      const double x1 = __ddiv_rn(rint(__dmul_rn(row[0], 100.0)), 100.0);
      const double y1 = __ddiv_rn(rint(__dmul_rn(row[1], 100.0)), 100.0);
      const double x2 = __ddiv_rn(rint(__dmul_rn(row[2], 100.0)), 100.0);
      const double y2 = __ddiv_rn(rint(__dmul_rn(row[3], 100.0)), 100.0);
      float c0, c1, s0, s1;
      rec_center_scale(x1, y1, x2, y2, aspect, my_bits, c0, c1, s0, s1);
      float src[6], dst[6];
      double m[6];
      rec_triangles(c0, c1, s0, ow, oh, src, dst);
      rec_affine(src, dst, m);
      bool finite = true;
      const long long r = at + p;
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        finite &= isfinite(m[i]);
        fwd_out[6 * r + i] = m[i];
      }
      if (!finite) my_bits |= REC_ST_MATRIX;
      frame_out[r] = (int)fr;
      slot_out[r] = (long long)rank * num_person + p;
      reinterpret_cast<float4*>(cs_out)[r] = make_float4(c0, c1, s0, s1);
    }
    // the tile's status bits and its first frame with a bit that names one
    int my_first = (my_bits & REC_ST_FRAME) ? t : K;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      my_bits |= __shfl_xor_sync(0xffffffffu, my_bits, o);
      my_first = min(my_first, __shfl_xor_sync(0xffffffffu, my_first, o));
    }
    if (lane == 0) {
      sh_red[warp][1] = my_bits;
      sh_red[warp][2] = my_first;
    }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < REC_WARPS; ++w) {
      bits |= sh_red[w][1];
      first = min(first, sh_red[w][2]);
    }
    __syncthreads();
    rec_done += tile.x;
    kept_done += tile.y;
  }
  if (tid == 0) {
    int* o = summary + 4 * s;
    o[0] = (int)rec_done;
    o[1] = kept_done;
    o[2] = bits | status[s];
    o[3] = first < K ? first : -1;
    if (s == S - 1) *total_out = (int)(base + rec_done);
  }
}

__global__ void __launch_bounds__(REC_INV_THREADS)
record_inverse_kernel(const float* __restrict__ cs, int n, const int* __restrict__ total, int hw, int hh,
                      double* __restrict__ out) {
  const int r = blockIdx.x * REC_INV_THREADS + threadIdx.x;
  if (r >= n || (total && r >= *total)) return;
  const float4 c = reinterpret_cast<const float4*>(cs)[r];
  float src[6], dst[6];
  double m[6];
  rec_triangles(c.x, c.y, c.z, hw, hh, src, dst);
  rec_affine(dst, src, m);
#pragma unroll
  for (int i = 0; i < 6; ++i) out[6 * (long long)r + i] = m[i];
}

}  // namespace gast

extern "C" int gast_track_records(const double* rows, const int32_t* counts, const int32_t* status, int32_t S,
                                  int32_t K, int32_t capacity, int32_t num_person, int32_t W, int32_t H, int32_t out_w,
                                  int32_t out_h, int32_t* frame_index, int64_t* slots, double* forward_mats,
                                  float* center_scale, int32_t* summary, int32_t* total, void* stream) {
  using namespace gast;
  if (!rows || !counts || !status || !frame_index || !slots || !forward_mats || !center_scale || !summary || !total ||
      S < 0 || K < 0 || capacity < 1 || num_person < 1)
    return fail("gast_track_records: bad arguments");
  if (W < 1 || H < 1 || W > REC_MAX_SIDE || H > REC_MAX_SIDE)
    return fail("gast_track_records: a %d x %d frame (each side 1 .. %d)", W, H, REC_MAX_SIDE);
  if (out_w < 1 || out_h < 1 || out_w > REC_MAX_SIDE || out_h > REC_MAX_SIDE)
    return fail("gast_track_records: a %d x %d crop (each side 1 .. %d)", out_w, out_h, REC_MAX_SIDE);
  if ((long long)S * K * num_person > 0x7fffffffLL)
    return fail("gast_track_records: %d x %d frames of %d persons exceed 2^31 - 1 records", S, K, num_person);
  if (S == 0) return 0;
  track_records_kernel<<<S, REC_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      rows, counts, status, K, capacity, num_person, W, H, out_w, out_h, S, frame_index,
      reinterpret_cast<long long*>(slots), forward_mats, center_scale, summary, total);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_record_inverse(const float* center_scale, int32_t n, const int32_t* total, int32_t hw, int32_t hh,
                                   double* inverse_mats, void* stream) {
  using namespace gast;
  if (!center_scale || !inverse_mats || n < 0) return fail("gast_record_inverse: bad arguments");
  if (hw < 1 || hh < 1 || hw > REC_MAX_SIDE || hh > REC_MAX_SIDE)
    return fail("gast_record_inverse: a %d x %d heatmap (each side 1 .. %d)", hw, hh, REC_MAX_SIDE);
  if (n == 0) return 0;
  record_inverse_kernel<<<cdiv(n, REC_INV_THREADS), REC_INV_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      center_scale, n, total, hw, hh, inverse_mats);
  CUDA_OK(cudaGetLastError());
  return 0;
}
