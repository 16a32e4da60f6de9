// The two data-parallel steps either side of the 2D pose net (lib/pose/hrnet/pose_estimation/gen_kpts.py:234-256):
//   gast_person_crops   PreProcess's crops (utils/utilitys.py:140-170): cv2.warpAffine(frame, M, (w, h), INTER_LINEAR)
//                       with a constant 0 border, then ToTensor and Normalize, for many boxes of many frames at once;
//   gast_heatmap_decode get_final_preds (utils/inference.py:21-82): argmax, the quarter-pixel shift and the inverse
//                       affine of every heatmap.
//
// The crop restates OpenCV's fixed-point bilinear warp (imgwarp.cpp's WarpAffineInvoker and remapBilinear): the
// matrix inverted in double, source coordinates in 1/32 pixel from rounded 1/1024 steps, integer weights summing to
// 32768.  One thread owns one output pixel and writes its three planes; nothing is shared and nothing is summed
// across threads, so a crop's bytes do not depend on the other records of the call and calls repeat bit for bit.
// The decode gives each (record, joint) heatmap one warp, with a fixed butterfly over a total order (value, then
// index), so its result does not depend on the launch either.  Every float operation is an explicit round-to-nearest
// intrinsic, in the order DESIGN.md §8.6 writes down; tests/keypoints2dref.py restates both kernels in numpy.
//
// Included at the end of gast_api.cu (uses fail / CUDA_OK / cdiv).
#pragma once
#include <math.h>

namespace gast {

constexpr int KP2D_MAX_SIDE = 32767;     // OpenCV keeps source coordinates as int16
constexpr int KP2D_MAX_HEATMAP = 256;    // heatmap side
constexpr int KP2D_MAX_J = 32;
constexpr int KP2D_CROP_THREADS = 256;
constexpr int KP2D_DECODE_WARPS = 8;

// transforms.Normalize's statistics as torch holds them: the float32 roundings of the Python doubles
__constant__ float kp2d_mean[3] = {static_cast<float>(0.485), static_cast<float>(0.456), static_cast<float>(0.406)};
__constant__ float kp2d_std[3] = {static_cast<float>(0.229), static_cast<float>(0.224), static_cast<float>(0.225)};

__device__ __forceinline__ int kp2d_short(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

// blockIdx.y strides over the records, blockIdx.x over the crop's pixels
__global__ void __launch_bounds__(KP2D_CROP_THREADS)
person_crop_kernel(const unsigned char* __restrict__ frames, long long n_frames, int H, int W,
                   const int* __restrict__ frame_index, const double* __restrict__ mats, int n, int ow, int oh,
                   int rgb_input, int net_order, float* __restrict__ out) {
  const int pix = blockIdx.x * KP2D_CROP_THREADS + threadIdx.x;
  if (pix >= ow * oh) return;
  const int x = pix % ow, y = pix / ow;
  const long long plane = (long long)ow * oh;
  for (int r = blockIdx.y; r < n; r += gridDim.y) {
    // the forward matrix inverted as warpAffine does it
    const double* m = mats + 6 * (long long)r;
    double M0 = m[0], M1 = m[1], M2 = m[2], M3 = m[3], M4 = m[4], M5 = m[5];
    double D = __dsub_rn(__dmul_rn(M0, M4), __dmul_rn(M1, M3));
    D = D != 0.0 ? __ddiv_rn(1.0, D) : 0.0;
    const double A11 = __dmul_rn(M4, D), A22 = __dmul_rn(M0, D);
    M0 = A11;
    M1 = __dmul_rn(M1, -D);
    M3 = __dmul_rn(M3, -D);
    M4 = A22;
    const double b1 = __dsub_rn(__dmul_rn(-M0, M2), __dmul_rn(M1, M5));
    const double b2 = __dsub_rn(__dmul_rn(-M3, M2), __dmul_rn(M4, M5));

    // fixed point: 1/1024 steps rounded half to even, then 1/32 pixel
    const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(M0, (double)x), 1024.0));
    const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(M3, (double)x), 1024.0));
    const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(M1, (double)y), b1), 1024.0)) + 16;
    const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(M4, (double)y), b2), 1024.0)) + 16;
    const int X = (int)((unsigned)X0 + (unsigned)adelta) >> 5;
    const int Y = (int)((unsigned)Y0 + (unsigned)bdelta) >> 5;
    const int sx = kp2d_short(X >> 5), sy = kp2d_short(Y >> 5), fx = X & 31, fy = Y & 31;
    const int w[4] = {(32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32};

    const long long f = frame_index[r];
    const bool have = f >= 0 && f < n_frames;
    const unsigned char* img = frames + f * H * W * 3;
    int acc[3] = {16384, 16384, 16384};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int xx = sx + (k & 1), yy = sy + (k >> 1);
      if (have && xx >= 0 && xx < W && yy >= 0 && yy < H) {
        const unsigned char* p = img + ((long long)yy * W + xx) * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += w[k] * (int)p[c];
      }
    }
    // plane c of the reference's order is the frame's BGR channel c, normalised with statistics c
    float* o = out + (long long)r * 3 * plane + pix;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int v8 = min(max(acc[rgb_input ? 2 - c : c] >> 15, 0), 255);
      const float v = __fdiv_rn((float)v8, 255.f);
      o[(net_order ? 2 - c : c) * plane] = __fdiv_rn(__fsub_rn(v, kp2d_mean[c]), kp2d_std[c]);
    }
  }
}

// np.argmax / np.amax order: a NaN beats every number and the first NaN wins; otherwise the larger value, and the
// smaller index among equals.  idx < 0 is the empty candidate.
__device__ __forceinline__ bool kp2d_beats(float v, int i, float bv, int bi) {
  if (i < 0) return false;
  if (bi < 0) return true;
  const bool vn = isnan(v), bn = isnan(bv);
  if (vn || bn) return vn && (!bn || i < bi);
  return v > bv || (v == bv && i < bi);
}

__global__ void __launch_bounds__(KP2D_DECODE_WARPS * 32)
heatmap_decode_kernel(const float* __restrict__ hm, const double* __restrict__ inv, int n, int J, int hh, int hw,
                      int post_process, float* __restrict__ preds, float* __restrict__ maxvals) {
  const long long wid = (long long)blockIdx.x * KP2D_DECODE_WARPS + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (wid >= (long long)n * J) return;
  const int S = hh * hw;
  const float* map = hm + wid * S;

  float bv = 0.f;
  int bi = -1;
#pragma unroll 4
  for (int i = lane; i < S; i += 32) {
    const float v = __ldg(map + i);
    if (bi < 0 || (!isnan(bv) && (isnan(v) || v > bv))) { bv = v; bi = i; }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, s);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, s);
    if (kp2d_beats(ov, oi, bv, bi)) { bv = ov; bi = oi; }
  }
  if (lane != 0) return;

  // get_max_preds: the index as float32, masked by maxval > 0 (false for NaN)
  const float mask = bv > 0.f ? 1.f : 0.f;
  float x = __fmul_rn((float)(bi % hw), mask);
  float y = __fmul_rn(floorf(__fdiv_rn((float)bi, (float)hw)), mask);
  if (post_process) {
    const int px = (int)floorf(__fadd_rn(x, 0.5f)), py = (int)floorf(__fadd_rn(y, 0.5f));
    if (1 < px && px < hw - 1 && 1 < py && py < hh - 1) {
      const float dx = __fsub_rn(map[py * hw + px + 1], map[py * hw + px - 1]);
      const float dy = __fsub_rn(map[(py + 1) * hw + px], map[(py - 1) * hw + px]);
      // np.sign: -1, 0 or 1, and NaN for NaN (then the coordinate is NaN)
      const float sx = dx > 0.f ? 1.f : (dx < 0.f ? -1.f : __fmul_rn(dx, 0.f));
      const float sy = dy > 0.f ? 1.f : (dy < 0.f ? -1.f : __fmul_rn(dy, 0.f));
      x = __fadd_rn(x, __fmul_rn(sx, 0.25f));
      y = __fadd_rn(y, __fmul_rn(sy, 0.25f));
    }
  }
  // transform_preds: np.dot(inverse, [x, y, 1]) in double as numpy's BLAS evaluates it, stored into float32
  const double* m = inv + 6 * (wid / J);
  const double xd = x, yd = y;
  preds[2 * wid] = __double2float_rn(__dadd_rn(__fma_rn(m[0], xd, __dmul_rn(m[1], yd)), m[2]));
  preds[2 * wid + 1] = __double2float_rn(__dadd_rn(__fma_rn(m[3], xd, __dmul_rn(m[4], yd)), m[5]));
  maxvals[wid] = bv;
}

}  // namespace gast

extern "C" int gast_person_crops(const uint8_t* frames, int64_t n_frames, int32_t H, int32_t W,
                                 const int32_t* frame_index, const double* forward_mats, int32_t n, int32_t out_w,
                                 int32_t out_h, int32_t flags, float* out, void* stream) {
  using namespace gast;
  if (!frames || !frame_index || !forward_mats || !out || n_frames <= 0 || n < 0 || flags < 0 || flags > 3)
    return fail("gast_person_crops: bad arguments (flags: GAST_CROP_RGB_INPUT | GAST_CROP_NET_ORDER)");
  if (H <= 0 || W <= 0 || H > KP2D_MAX_SIDE || W > KP2D_MAX_SIDE)
    return fail("gast_person_crops: a %d x %d frame (each side 1 .. %d)", W, H, KP2D_MAX_SIDE);
  if (out_w <= 0 || out_h <= 0 || out_w > KP2D_MAX_SIDE || out_h > KP2D_MAX_SIDE)
    return fail("gast_person_crops: a %d x %d crop (each side 1 .. %d)", out_w, out_h, KP2D_MAX_SIDE);
  if (n == 0) return 0;
  const dim3 grid(cdiv((long long)out_w * out_h, KP2D_CROP_THREADS), (unsigned)min(n, 65535));
  person_crop_kernel<<<grid, KP2D_CROP_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      frames, n_frames, H, W, frame_index, forward_mats, n, out_w, out_h, flags & 1, (flags >> 1) & 1, out);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_heatmap_decode(const float* heatmaps, const double* inverse_mats, int32_t n, int32_t J,
                                   int32_t hh, int32_t hw, int32_t post_process, float* preds, float* maxvals,
                                   void* stream) {
  using namespace gast;
  if (!heatmaps || !inverse_mats || !preds || !maxvals || n < 0 || (post_process != 0 && post_process != 1))
    return fail("gast_heatmap_decode: bad arguments");
  if (J < 1 || J > KP2D_MAX_J || hh < 1 || hw < 1 || hh > KP2D_MAX_HEATMAP || hw > KP2D_MAX_HEATMAP)
    return fail("gast_heatmap_decode: %d joints of %d x %d heatmaps (J <= %d, sides <= %d)", J, hw, hh, KP2D_MAX_J,
                KP2D_MAX_HEATMAP);
  if (n == 0) return 0;
  heatmap_decode_kernel<<<cdiv((long long)n * J, KP2D_DECODE_WARPS), KP2D_DECODE_WARPS * 32, 0,
                          reinterpret_cast<cudaStream_t>(stream)>>>(heatmaps, inverse_mats, n, J, hh, hw, post_process,
                                                                     preds, maxvals);
  CUDA_OK(cudaGetLastError());
  return 0;
}
