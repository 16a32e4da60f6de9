// The person detector's data-parallel steps either side of Darknet (lib/detector/yolov3/human_detector.py:106-157):
//   gast_letterbox           preprocess.prep_image of many frames: letterbox_image's cv2.resize(INTER_CUBIC) pasted
//                            into a 128 canvas, BGR -> RGB, /255;
//   gast_person_detections   util.write_results(det_hm=True) (confidence mask, corners, class argmax, person filter,
//                            sort, greedy NMS) and yolo_human_det's rescale, clamp and round, per frame.
//
// The letterbox restates OpenCV's own INTER_CUBIC path for uint8 (resize.cpp: resizeGeneric_ with HResizeCubic and
// VResizeCubic): interpolateCubic's float coefficients as 11-bit shorts, the horizontal pass in int32 with the edge
// clamped, and the vertical pass as OpenCV's 128-bit vector loop computes it (float32 multiply-adds, rounded half to
// even) for the first 8 * floor(3 new_w / 8) interleaved values of a row, FixedPtCast<int, uchar, 22> for the rest.
// One thread owns one canvas pixel and writes its three planes.
//
// The post-processing gives each frame one CTA: it filters the frame's rows (objectness first, the 80 class scores
// only for rows that pass), compacts the candidates in row order by block scans, sorts them in shared memory on a
// 64-bit key (objectness descending, NaN first, then the row: the one place where the device fixes an order the
// reference leaves open), runs the greedy NMS as one block-wide pass per surviving row, and writes the survivors.
// Nothing is ordered by atomics, so calls repeat bit for bit.  Every float operation is an explicit round-to-nearest
// intrinsic in the order DESIGN.md §8.7 writes down; tests/detectionref.py restates both kernels in numpy.
//
// Included at the end of gast_api.cu (uses fail / CUDA_OK / cdiv).
#pragma once
#include <math.h>

namespace gast {

constexpr int DET_MAX_SIDE = 32767;        // OpenCV's resize keeps coordinates as int
constexpr int DET_ATTRS = 85;              // x, y, w, h, objectness, 80 class scores
constexpr int DET_CLASSES = 80;
constexpr int DET_LB_THREADS = 256;
constexpr int DET_NMS_THREADS = 512;
constexpr int DET_SIMD_STEP = 8;           // interleaved values per step of OpenCV's vertical vector loop
constexpr int DET_MAX_SMEM = 227 * 1024;   // opt-in shared memory per block on sm_90

// interpolateCubic (A = -0.75) in float32 with its last coefficient 1 - the others, as saturate_cast<short>(c * 2048)
__device__ __forceinline__ void det_cubic(float x, int c[4]) {
  const float A = -0.75f;
  const float x1 = __fadd_rn(x, 1.f);
  const float c0 = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), -3.75f), x1), -6.f), x1), -3.f);
  const float c1 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, x), 2.25f), x), x), 1.f);
  const float om = __fsub_rn(1.f, x);
  const float c2 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(1.25f, om), 2.25f), om), om), 1.f);
  const float c3 = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c0), c1), c2);
  const float cf[4] = {c0, c1, c2, c3};
#pragma unroll
  for (int k = 0; k < 4; ++k) c[k] = min(max(__float2int_rn(__fmul_rn(cf[k], 2048.f)), -32768), 32767);
}

// one axis: the first of the four source taps (before clamping) and the coefficients of destination index d
__device__ __forceinline__ int det_axis(int d, double scale, int c[4]) {
  const float f = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
  const float s = floorf(f);
  det_cubic(__fsub_rn(f, s), c);
  return (int)s - 1;
}

// blockIdx.y strides over the frames, blockIdx.x over the canvas pixels
__global__ void __launch_bounds__(DET_LB_THREADS)
letterbox_kernel(const unsigned char* __restrict__ frames, int n, int H, int W, int D, int nw, int nh, int ox, int oy,
                 double scale_x, double scale_y, int rgb_input, float* __restrict__ out) {
  const int pix = blockIdx.x * DET_LB_THREADS + threadIdx.x;
  if (pix >= D * D) return;
  const int x = pix % D, y = pix / D;
  const long long plane = (long long)D * D;
  const int dx = x - ox, dy = y - oy;
  const bool inside = dx >= 0 && dx < nw && dy >= 0 && dy < nh;
  int cx[4], cy[4], xs[4], ys[4];
  if (inside) {
    const int sx = det_axis(dx, scale_x, cx), sy = det_axis(dy, scale_y, cy);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      xs[k] = min(max(sx + k, 0), W - 1);
      ys[k] = min(max(sy + k, 0), H - 1);
    }
  }
  const int nvec = (3 * nw / DET_SIMD_STEP) * DET_SIMD_STEP;
  const float inv_scale = 1.f / (2048.f * 2048.f);
  for (int f = blockIdx.y; f < n; f += gridDim.y) {
    float* o = out + (long long)f * 3 * plane + pix;
    if (!inside) {
#pragma unroll
      for (int p = 0; p < 3; ++p) o[p * plane] = __fdiv_rn(128.f, 255.f);
      continue;
    }
    const unsigned char* img = frames + (long long)f * H * W * 3;
    // the horizontal pass of the four source rows, per BGR channel of the resized image
    int hs[4][3];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const unsigned char* row = img + (long long)ys[r] * W * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int src_c = rgb_input ? 2 - c : c;
        int v = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) v += (int)__ldg(row + xs[k] * 3 + src_c) * cx[k];
        hs[r][c] = v;
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      int v8;
      if (3 * dx + c < nvec) {
        float t = __fmul_rn((float)hs[3][c], __fmul_rn((float)cy[3], inv_scale));
#pragma unroll
        for (int k = 2; k >= 0; --k) t = __fadd_rn(__fmul_rn((float)hs[k][c], __fmul_rn((float)cy[k], inv_scale)), t);
        v8 = __float2int_rn(t);
      } else {
        const int s = hs[0][c] * cy[0] + hs[1][c] * cy[1] + hs[2][c] * cy[2] + hs[3][c] * cy[3];
        v8 = (s + (1 << 21)) >> 22;
      }
      v8 = min(max(v8, 0), 255);
      // plane 0 is R: BGR channel 2
      o[(2 - c) * plane] = __fdiv_rn((float)v8, 255.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// post-processing
// ------------------------------------------------------------------------------------------------
// torch.max / torch.min of two float32 tensors: NaN if either is NaN
__device__ __forceinline__ float det_tmax(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : (a < b ? b : a); }
__device__ __forceinline__ float det_tmin(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fc00000) : (b < a ? b : a); }

// bbox_iou of two corner boxes with its +1 areas
__device__ __forceinline__ float det_iou(float4 a, float4 b) {
  const float ix1 = det_tmax(a.x, b.x), iy1 = det_tmax(a.y, b.y);
  const float ix2 = det_tmin(a.z, b.z), iy2 = det_tmin(a.w, b.w);
  const float inter = __fmul_rn(det_tmax(__fadd_rn(__fsub_rn(ix2, ix1), 1.f), 0.f),
                                det_tmax(__fadd_rn(__fsub_rn(iy2, iy1), 1.f), 0.f));
  const float a1 = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.f), __fadd_rn(__fsub_rn(a.w, a.y), 1.f));
  const float a2 = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(a1, a2), inter));
}

// the confidence mask: 1 for obj > conf, else 0 (the row is multiplied by it)
__device__ __forceinline__ float det_mask(float obj, float conf) { return obj > conf ? 1.f : 0.f; }

// a row's corners after the mask: x - w/2, y - h/2, x + w/2, y + h/2; zeroed (each value * 0) by a suppression
__device__ __forceinline__ float4 det_box(const float* p, float m, bool zeroed) {
  const float x = __fmul_rn(p[0], m), y = __fmul_rn(p[1], m);
  const float hw = __fdiv_rn(__fmul_rn(p[2], m), 2.f), hh = __fdiv_rn(__fmul_rn(p[3], m), 2.f);
  float4 b = make_float4(__fsub_rn(x, hw), __fsub_rn(y, hh), __fadd_rn(x, hw), __fadd_rn(y, hh));
  if (zeroed) b = make_float4(__fmul_rn(b.x, 0.f), __fmul_rn(b.y, 0.f), __fmul_rn(b.z, 0.f), __fmul_rn(b.w, 0.f));
  return b;
}

// 0 not a candidate, 1 a person row that max_conf == 0 drops, 2 a candidate.  obj * mask must be nonzero (NaN is),
// the class argmax (first maximum, the first NaN winning) must be class 0 and its masked score nonzero.
__device__ __forceinline__ int det_classify(const float* p, float conf, float* obj_out) {
  const float obj = __ldg(p + 4);
  const float m = det_mask(obj, conf);
  const float o = __fmul_rn(obj, m);
  *obj_out = o;
  if (o == 0.f) return 0;
  const float s0 = __fmul_rn(__ldg(p + 5), m);
  if (s0 == s0) {
    for (int k = 1; k < DET_CLASSES; ++k) {
      const float s = __fmul_rn(__ldg(p + 5 + k), m);
      if (s != s || s0 < s) return 0;
    }
  }
  return s0 != 0.f ? 2 : 1;
}

// the sort key: ascending order of ((~sortable(obj)) << 32 | row) is objectness descending (NaN first), then row
__device__ __forceinline__ unsigned long long det_key(float obj, int row) {
  unsigned u = __float_as_uint(obj);
  u = (obj != obj) ? 0xffffffffu : ((u & 0x80000000u) ? ~u : (u | 0x80000000u));
  return ((unsigned long long)(~u) << 32) | (unsigned)row;
}

// exclusive block scan of one flag per thread; returns the thread's offset, *total the block's count
__device__ __forceinline__ int det_block_scan(int flag, int* warp_sums, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const unsigned ball = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_sums[warp] = __popc(ball);
  __syncthreads();
  if (warp == 0) {
    const int v = lane < nwarps ? warp_sums[lane] : 0;
    int s = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += t;
    }
    if (lane < nwarps) warp_sums[lane] = s - v;
    if (lane == 31) warp_sums[32] = s;
  }
  __syncthreads();
  const int off = warp_sums[warp] + __popc(ball & ((1u << lane) - 1u));
  *total = warp_sums[32];
  __syncthreads();
  return off;
}

// shared memory: N 64-bit keys, then N state bytes (1 alive, 2 alive with its box zeroed, 0 suppressed)
__global__ void __launch_bounds__(DET_NMS_THREADS)
person_detections_kernel(const float* __restrict__ pred, int N, int D, const int* __restrict__ sizes, float conf,
                         float nms_thresh, int max_det, int raw, float* __restrict__ boxes, float* __restrict__ scores,
                         int* __restrict__ counts, float* __restrict__ max_conf, int* __restrict__ persons) {
  extern __shared__ unsigned long long det_keys[];
  unsigned char* state = reinterpret_cast<unsigned char*>(det_keys + N);
  __shared__ int warp_sums[33];
  const int f = blockIdx.x;
  const float* P = pred + (long long)f * N * DET_ATTRS;

  // 1. the candidates, compacted in row order
  int n = 0, person_rows = 0;
  for (int base = 0; base < N; base += blockDim.x) {
    const int row = base + threadIdx.x;
    float obj = 0.f;
    const int cls = row < N ? det_classify(P + (long long)row * DET_ATTRS, conf, &obj) : 0;
    person_rows += __syncthreads_count(cls != 0);
    int total;
    const int off = det_block_scan(cls == 2, warp_sums, &total);
    if (cls == 2) {
      det_keys[n + off] = det_key(obj, row);
      state[n + off] = 1;
    }
    n += total;
  }

  // 2. sort: a bitonic network whose comparators all put the smaller key first, so the virtual +inf keys past n
  // never move and only n keys are stored
  int P2 = 1;
  while (P2 < n) P2 <<= 1;
  for (int k = 2; k <= P2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < (P2 >> 1); t += blockDim.x) {
        int a, b;
        if (j == (k >> 1)) {
          const int blk = t / j, off = t % j;
          a = blk * k + off;
          b = blk * k + k - 1 - off;
        } else {
          const int blk = t / j, off = t % j;
          a = blk * 2 * j + off;
          b = a + j;
        }
        if (b < n) {
          const unsigned long long ka = det_keys[a], kb = det_keys[b];
          if (kb < ka) {
            det_keys[a] = kb;
            det_keys[b] = ka;
          }
        }
      }
    }
  }
  __syncthreads();

  // 3. greedy NMS: each surviving row, in order, multiplies the later rows by (iou < nms_thresh); a row whose
  // objectness becomes 0 goes, a non-finite one stays with its box zeroed
  for (int i = 0; i < n; ++i) {
    const unsigned char si = state[i];
    if (si == 0) continue;                          // uniform: state[i] is final once every row before it ran
    const int ri = (int)(det_keys[i] & 0xffffffffu);
    const float* pi = P + (long long)ri * DET_ATTRS;
    const float4 bi = det_box(pi, det_mask(pi[4], conf), si == 2);
    for (int k = i + 1 + threadIdx.x; k < n; k += blockDim.x) {
      const unsigned char sk = state[k];
      if (sk == 0) continue;
      const int rk = (int)(det_keys[k] & 0xffffffffu);
      const float* pk = P + (long long)rk * DET_ATTRS;
      const float mk = det_mask(pk[4], conf);
      if (!(det_iou(bi, det_box(pk, mk, sk == 2)) < nms_thresh))
        state[k] = __fmul_rn(__fmul_rn(pk[4], mk), 0.f) == 0.f ? 0 : 2;
    }
    __syncthreads();
  }

  // 4. the survivors in order: rescaled to the frame, clamped and rounded to 2 decimals (or write_results' corners)
  const float W = (float)sizes[2 * f], H = (float)sizes[2 * f + 1], Df = (float)D;
  const float sf = fminf(__fmul_rn(__frcp_rn(W), Df), __fmul_rn(__frcp_rn(H), Df));
  const float px = __fdiv_rn(__fsub_rn(Df, __fmul_rn(sf, W)), 2.f);
  const float py = __fdiv_rn(__fsub_rn(Df, __fmul_rn(sf, H)), 2.f);
  int written = 0;
  for (int base = 0; base < n; base += blockDim.x) {
    const int s = base + threadIdx.x;
    const unsigned char st = s < n ? state[s] : 0;
    int total;
    const int off = det_block_scan(st != 0, warp_sums, &total);
    const int slot = written + off;
    if (st != 0 && slot < max_det) {
      const int r = (int)(det_keys[s] & 0xffffffffu);
      const float* p = P + (long long)r * DET_ATTRS;
      const float m = det_mask(p[4], conf);
      const bool zeroed = st == 2;
      float4 b = det_box(p, m, zeroed);
      if (!raw) {
        float v[4] = {__fdiv_rn(__fsub_rn(b.x, px), sf), __fdiv_rn(__fsub_rn(b.y, py), sf),
                      __fdiv_rn(__fsub_rn(b.z, px), sf), __fdiv_rn(__fsub_rn(b.w, py), sf)};
        const float lim[4] = {W, H, W, H};
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          float t = v[c] < 0.f ? 0.f : v[c];          // std::max(v, 0): NaN stays
          t = lim[c] < t ? lim[c] : t;                // std::min(v, lim)
          v[c] = __fdiv_rn(rintf(__fmul_rn(t, 100.f)), 100.f);
        }
        b = make_float4(v[0], v[1], v[2], v[3]);
      }
      const long long o = (long long)f * max_det + slot;
      reinterpret_cast<float4*>(boxes)[o] = b;
      float obj = __fmul_rn(p[4], m), s0 = __fmul_rn(p[5], m);
      if (zeroed) obj = __fmul_rn(obj, 0.f), s0 = __fmul_rn(s0, 0.f);
      scores[o] = obj;
      if (max_conf) max_conf[o] = s0;
    }
    written += total;
  }
  for (int slot = written + threadIdx.x; slot < max_det; slot += blockDim.x) {
    const long long o = (long long)f * max_det + slot;
    reinterpret_cast<float4*>(boxes)[o] = make_float4(0.f, 0.f, 0.f, 0.f);
    scores[o] = 0.f;
    if (max_conf) max_conf[o] = 0.f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    counts[f] = written;
    if (persons) persons[f] = person_rows;
  }
}

inline long long det_num_predictions(int D) { return 3LL * ((D / 32) * (D / 32) + (D / 16) * (D / 16) + (D / 8) * (D / 8)); }
inline size_t det_smem_bytes(long long N) { return (size_t)N * (sizeof(unsigned long long) + 1); }

}  // namespace gast

extern "C" int gast_letterbox(const uint8_t* frames, int32_t n, int32_t H, int32_t W, int32_t D, int32_t new_w,
                              int32_t new_h, int32_t flags, float* out, void* stream) {
  using namespace gast;
  if (!frames || !out || n < 0 || flags < 0 || flags > 1) return fail("gast_letterbox: bad arguments (flags: GAST_LETTERBOX_RGB_INPUT)");
  if (H <= 0 || W <= 0 || H > DET_MAX_SIDE || W > DET_MAX_SIDE)
    return fail("gast_letterbox: a %d x %d frame (each side 1 .. %d)", W, H, DET_MAX_SIDE);
  if (D <= 32 || D % 32 != 0) return fail("gast_letterbox: inp_dim %d (a multiple of 32 above 32)", D);
  if (new_w <= 0 || new_h <= 0 || new_w > D || new_h > D)
    return fail("gast_letterbox: a %d x %d resize into %d x %d", new_w, new_h, D, D);
  if (n == 0) return 0;
  // cv2.resize: inv_scale = (double)new / old, scale = 1 / inv_scale
  const double sx = 1.0 / ((double)new_w / W), sy = 1.0 / ((double)new_h / H);
  const dim3 grid(cdiv((long long)D * D, DET_LB_THREADS), (unsigned)min(n, 65535));
  letterbox_kernel<<<grid, DET_LB_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      frames, n, H, W, D, new_w, new_h, (D - new_w) / 2, (D - new_h) / 2, sx, sy, flags & 1, out);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_person_detections(const float* predictions, int32_t n, int32_t N, int32_t attrs, int32_t D,
                                      const int32_t* frame_sizes, float confidence, float nms_thresh, int32_t max_det,
                                      int32_t flags, float* boxes, float* scores, int32_t* counts, float* max_conf,
                                      int32_t* persons, void* stream) {
  using namespace gast;
  if (!predictions || !frame_sizes || !boxes || !scores || !counts || n < 0 || max_det < 0 || flags < 0 || flags > 1)
    return fail("gast_person_detections: bad arguments (flags: GAST_DETECT_RAW)");
  if (D <= 32 || D % 32 != 0) return fail("gast_person_detections: inp_dim %d (a multiple of 32 above 32)", D);
  if (attrs != DET_ATTRS) return fail("gast_person_detections: %d attributes per prediction (85 expected)", attrs);
  const long long want = det_num_predictions(D);
  if (N != want) return fail("gast_person_detections: %d predictions for inp_dim %d (%lld expected)", N, D, want);
  const size_t smem = det_smem_bytes(N);
  if (smem > (size_t)DET_MAX_SMEM)
    return fail("gast_person_detections: inp_dim %d: %lld predictions need %zu bytes of shared memory (at most %d)", D,
                want, smem, DET_MAX_SMEM);
  if (n == 0) return 0;
  CUDA_OK(cudaFuncSetAttribute(person_detections_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  person_detections_kernel<<<n, DET_NMS_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      predictions, N, D, frame_sizes, confidence, nms_thresh, max_det, flags & 1, boxes, scores, counts, max_conf,
      persons);
  CUDA_OK(cudaGetLastError());
  return 0;
}
