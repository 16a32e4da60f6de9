// The callers and data formats either side of the lifting forward (SURVEY.md §8f N1-N3), kept on the
// device: training-batch assembly (ChunkedGenerator), keypoint format conversion and screen
// normalisation in front of the network; camera-to-world, MPJPE / P-MPJPE and the optimiser step
// behind it.  All are HBM-/latency-bound elementwise or tiny-reduction kernels; what they buy is
// that a 200k clips/s forward is not fed and drained by numpy on the host.
//
// Included at the end of gast_api.cu (uses fail / CUDA_OK / cdiv / JointPerm / make_perm).
#pragma once
#include <algorithm>
#include <math.h>

namespace gast {

// ------------------------------------------------------------------------------------------
// N1: ChunkedGenerator.next_epoch (common/generators.py:93-154): one training batch gathered from
// the concatenated sequences.  pairs[b] = {seq, start_3d, end_3d (unused), flip}.
//   batch_2d[b,t] = edge-clamped frame (start_3d - pad - causal_shift + t) of sequence seq, mirrored
//   when flip (feature 0 negated, left/right keypoints swapped); batch_3d likewise without padding;
//   batch_cam[b] = cameras[seq] with entries 2 and 7 negated when flip (:139-144).
// ------------------------------------------------------------------------------------------
__global__ void chunk_gather_kernel(const float* __restrict__ poses, const long long* __restrict__ seq_start,
                                    const int* __restrict__ pairs, float* __restrict__ out, int B, int Tc, int J, int F,
                                    int lead, JointPerm perm) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long n = (long long)B * Tc * J * F;
  if (idx >= n) return;
  const int c = (int)(idx % F);
  const int j = (int)((idx / F) % J);
  const int t = (int)((idx / ((long long)F * J)) % Tc);
  const int b = (int)(idx / ((long long)F * J * Tc));
  const int seq = pairs[4 * b], start = pairs[4 * b + 1], flip = pairs[4 * b + 3];
  const long long s0 = seq_start[seq], len = seq_start[seq + 1] - s0;
  long long fr = (long long)start - lead + t;
  fr = fr < 0 ? 0 : (fr > len - 1 ? len - 1 : fr);              // np.pad(..., 'edge')
  const int js = flip ? perm.p[j] : j;
  float v = poses[((s0 + fr) * J + js) * F + c];
  out[idx] = (flip && c == 0) ? -v : v;
}

__global__ void chunk_cam_kernel(const float* __restrict__ cams, const int* __restrict__ pairs, float* __restrict__ out,
                                 int B, int ncam) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * ncam) return;
  const int b = idx / ncam, k = idx - b * ncam;
  float v = cams[(long long)pairs[4 * b] * ncam + k];
  if (pairs[4 * b + 3] && (k == 2 || k == 7)) v = -v;
  out[idx] = v;
}

// ------------------------------------------------------------------------------------------
// N3: keypoint formats (tools/mpii_coco_h36m.py).  One thread per frame; float32 arithmetic in the
// order numpy evaluates it (sequential sums, true division), so results are bit-identical for
// float32 input.  valid[t] = (sum of the frame's coordinates != 0), the mask np.where is taken of.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float np_pairwise_sum(const float* a, int n) {   // numpy's float32 add.reduce, 8 <= n < 128
  float r[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) r[k] = a[k];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
#pragma unroll
    for (int k = 0; k < 8; ++k) r[k] = __fadd_rn(r[k], a[i + k]);
  float res = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                        __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
  for (; i < n; ++i) res = __fadd_rn(res, a[i]);
  return res;
}

// coco_h36m (tools/mpii_coco_h36m.py:20-48): kp (17 x 2) of one frame -> h (17 x 2)
__device__ __forceinline__ void coco_to_h36m_frame(const float* kp, int ld, float* h) {
  auto K = [&](int j, int c) { return kp[j * ld + c]; };
  const int h36m_coco_order[13] = {9, 11, 14, 12, 15, 13, 16, 4, 1, 5, 2, 6, 3};
  const int coco_order[13] = {0, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
  float htps[4][2];
  htps[0][0] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(K(1, 0), K(2, 0)), K(3, 0)), K(4, 0)), 4.f);   // head x :25
  htps[0][1] = __fsub_rn(__fadd_rn(K(1, 1), K(2, 1)), K(0, 1));                                      // head y :26
#pragma unroll
  for (int c = 0; c < 2; ++c) {
    float th = __fdiv_rn(__fadd_rn(K(5, c), K(6, c)), 2.f);                                          // thorax :27
    th = __fadd_rn(th, __fdiv_rn(__fsub_rn(K(0, c), th), 3.f));                                      // :28
    htps[1][c] = th;
    htps[2][c] = __fdiv_rn(__fadd_rn(K(11, c), K(12, c)), 2.f);                                      // pelvis :30
    htps[3][c] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(K(5, c), K(6, c)), K(11, c)), K(12, c)), 4.f);   // spine :31
  }
  const int spple[4] = {10, 8, 0, 7};
#pragma unroll
  for (int i = 0; i < 4; ++i) { h[spple[i] * 2] = htps[i][0]; h[spple[i] * 2 + 1] = htps[i][1]; }
#pragma unroll
  for (int i = 0; i < 13; ++i) {
    h[h36m_coco_order[i] * 2] = K(coco_order[i], 0);
    h[h36m_coco_order[i] * 2 + 1] = K(coco_order[i], 1);
  }
#pragma unroll
  for (int c = 0; c < 2; ++c) {                                                                       // neck :36
    const float m = __fdiv_rn(__fadd_rn(K(5, c), K(6, c)), 2.f);
    h[9 * 2 + c] = __fsub_rn(h[9 * 2 + c], __fdiv_rn(__fsub_rn(h[9 * 2 + c], m), 4.f));
  }
  {                                                                                                   // spine x :37
    const float m = __fdiv_rn(__fadd_rn(h[0], h[8 * 2]), 2.f);
    h[7 * 2] = __fadd_rn(h[7 * 2], __fmul_rn(2.f, __fsub_rn(h[7 * 2], m)));
  }
  {                                                                                                   // thorax y :38
    const float m = __fdiv_rn(__fadd_rn(K(1, 1), K(2, 1)), 2.f);
    h[8 * 2 + 1] = __fsub_rn(h[8 * 2 + 1], __fdiv_rn(__fmul_rn(__fsub_rn(m, K(0, 1)), 2.f), 3.f));
  }
}

// mode 0: coco_h36m            kp (T,17,2)  -> out (T,17,2)
// mode 1: mpii_h36m            kp (T,16,2)  -> out (T,17,2)   (:51-59)
// mode 2: coco_h36m_toe_format kp (T,Jin>=22,2) -> out (T,19,2)   (:62-78)
__global__ void kpt_convert_kernel(const float* __restrict__ kp, float* __restrict__ out, int* __restrict__ valid,
                                   int T, int Jin, int mode) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const float* k = kp + (long long)t * Jin * 2;
  float o[38];
  int Jo = 17;
  if (mode == 0) {
    coco_to_h36m_frame(k, 2, o);
  } else if (mode == 1) {
    const int h36m_mpii_order[16] = {3, 2, 1, 4, 5, 6, 0, 8, 9, 10, 16, 15, 14, 11, 12, 13};
#pragma unroll
    for (int i = 0; i < 34; ++i) o[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) { o[h36m_mpii_order[i] * 2] = k[i * 2]; o[h36m_mpii_order[i] * 2 + 1] = k[i * 2 + 1]; }
#pragma unroll
    for (int c = 0; c < 2; ++c)
      o[7 * 2 + c] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(k[2 * 2 + c], k[3 * 2 + c]), k[12 * 2 + c]), k[13 * 2 + c]), 4.f);
  } else {
    Jo = 19;
    float h[34];
    coco_to_h36m_frame(k, 2, h);
    const int toe_order[17] = {0, 1, 2, 3, 5, 6, 7, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18};
#pragma unroll
    for (int i = 0; i < 38; ++i) o[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 17; ++i) { o[toe_order[i] * 2] = h[i * 2]; o[toe_order[i] * 2 + 1] = h[i * 2 + 1]; }
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      o[4 * 2 + c] = __fdiv_rn(__fadd_rn(k[20 * 2 + c], k[21 * 2 + c]), 2.f);
      o[8 * 2 + c] = __fdiv_rn(__fadd_rn(k[17 * 2 + c], k[18 * 2 + c]), 2.f);
    }
  }
  float* op = out + (long long)t * Jo * 2;
  for (int i = 0; i < Jo * 2; ++i) op[i] = o[i];
  if (valid) valid[t] = (np_pairwise_sum(o, Jo * 2) != 0.f) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------
// The video demo's keypoint repair and placement of the lifted persons (tools/preprocess.py), float32 in the
// reference's order of operations, so results are bit-identical for float32 input.
// ------------------------------------------------------------------------------------------
constexpr int PREP_BLOCK = 256;
__device__ __forceinline__ float np_minf(float a, float b) { return (isnan(a) || a < b) ? a : b; }   // np.amin: NaN wins

// h36m_coco_format (preprocess.py:47-75): one thread per (person, frame).  Keypoints and valid mask as
// kpt_convert_kernel mode 0; the scores remapped (:65-69); keep[p] = 1 once any coordinate of person p is non-zero
// (keep is zeroed by the caller; every writer stores the same value).
__global__ void h36m_coco_format_kernel(const float* __restrict__ kp, const float* __restrict__ sc, float* __restrict__ out,
                                        float* __restrict__ sout, int* __restrict__ valid, int* __restrict__ keep, int P,
                                        int T) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)P * T) return;
  const float* k = kp + i * 34;
  bool any = false;
  for (int c = 0; c < 34; ++c) any |= (k[c] != 0.f);
  if (any) keep[i / T] = 1;
  float o[34];
  coco_to_h36m_frame(k, 2, o);
  float* op = out + i * 34;
  for (int c = 0; c < 34; ++c) op[c] = o[c];
  valid[i] = (np_pairwise_sum(o, 34) != 0.f) ? 1 : 0;
  const float* s = sc + i * 17;
  float n[17];
  const int h36m_coco_order[13] = {9, 11, 14, 12, 15, 13, 16, 4, 1, 5, 2, 6, 3};
  const int coco_order[13] = {0, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16};
#pragma unroll
  for (int q = 0; q < 13; ++q) n[h36m_coco_order[q]] = s[coco_order[q]];
  n[0] = __fdiv_rn(__fadd_rn(s[11], s[12]), 2.f);
  n[8] = __fdiv_rn(__fadd_rn(s[5], s[6]), 2.f);
  n[7] = __fdiv_rn(__fadd_rn(n[0], n[8]), 2.f);
  n[10] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(s[1], s[2]), s[3]), s[4]), 4.f);
  float* so = sout + i * 17;
#pragma unroll
  for (int q = 0; q < 17; ++q) so[q] = n[q];
}

// revise_kpts (preprocess.py:78-112): one thread per (person, frame).  Zero outside the valid frames; at a valid
// frame the pose, with the low-confidence limb joints replaced by the first matching case of :94-109 (every right-hand
// side read before the assignment, as numpy's fancy indexing does).  low joints: score < float32(0.3).
__global__ void revise_kpts_kernel(const float* __restrict__ kp, const float* __restrict__ sc, const int* __restrict__ mask,
                                   float* __restrict__ out, long long PT, int J) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= PT) return;
  const float2* k = reinterpret_cast<const float2*>(kp) + i * J;
  float2* o = reinterpret_cast<float2*>(out) + i * J;
  if (!mask[i]) {
    for (int j = 0; j < J; ++j) o[j] = make_float2(0.f, 0.f);
    return;
  }
  for (int j = 0; j < J; ++j) o[j] = k[j];
  const float* s = sc + i * J;
  const int low = (s[2] < 0.3f ? 1 : 0) | (s[3] < 0.3f ? 2 : 0) | (s[5] < 0.3f ? 4 : 0) | (s[6] < 0.3f ? 8 : 0);
  const float2 k1 = k[1], k2 = k[2], k4 = k[4], k5 = k[5];
  switch (low) {
    case 15: o[2] = k1; o[3] = k1; o[5] = k4; o[6] = k4; break;   // [2, 3, 5, 6] <- [1, 1, 4, 4]
    case 11: o[2] = k1; o[3] = k1; o[6] = k5; break;              // [2, 3, 6] <- [1, 1, 5]
    case 14: o[3] = k2; o[5] = k4; o[6] = k4; break;              // [3, 5, 6] <- [2, 4, 4]
    case 10: o[3] = k2; o[6] = k5; break;                         // [3, 6] <- [2, 5]
    case 2: o[3] = k2; break;                                     // 3 <- 2
    case 8: o[6] = k5; break;                                     // 6 <- 5
    default: break;                                               // any other combination: unchanged
  }
}

// mean over joints [1, 4, 11, 14] of (a - b) (b may be null = 0), channel c of rows with D floats per joint:
// float32, left to right, then / 4 (np.mean over a 4-row axis)
__device__ __forceinline__ float limb_mean(const float* a, const float* b, int D, int c) {
  const int jj[4] = {1, 4, 11, 14};
  float s = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float v = b ? __fsub_rn(a[jj[q] * D + c], b[jj[q] * D + c]) : a[jj[q] * D + c];
    s = q == 0 ? v : __fadd_rn(s, v);
  }
  return __fdiv_rn(s, 4.f);
}

// revise_skes, two persons (:138-141): the first entry k of person 0's frames that person 1 also has (mask1 = person
// 1's valid mask); per block the smallest such k, INT_MAX when none.
__global__ void first_common_kernel(const long long* __restrict__ frames0, int F0, const int* __restrict__ mask1,
                                    int* __restrict__ part) {
  int best = INT_MAX;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < F0; k += gridDim.x * blockDim.x)
    if (mask1[frames0[k]]) best = min(best, k);
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  __shared__ int sh[PREP_BLOCK / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < PREP_BLOCK / 32; ++w) best = min(best, sh[w]);
    part[blockIdx.x] = best;
  }
}

__global__ void mask_scatter_kernel(const long long* __restrict__ frames, int F, int* __restrict__ mask) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < F) mask[frames[k]] = 1;
}

// revise_skes (:123-147): grid.y = person; one thread per (packed row, joint) of that person.  Scatters the packed
// prediction row k to frame frames[k]; rows after the first move by the limb-mean 2D displacement from the first
// valid frame / 500 (:130-133); with two persons both move by half their limb-mean distance at the first common frame
// (:138-147; ncommon_part blocks of first_common_kernel partials, NaN poses when there is no common frame).
// out must be zero.
__global__ void revise_skes_kernel(const float* __restrict__ pred, const long long* __restrict__ frames,
                                   const long long* __restrict__ off, const float* __restrict__ kp, float* __restrict__ out,
                                   int T, int J, int D, const int* __restrict__ common_part, int ncommon_part) {
  const int p = blockIdx.y;
  const long long o0 = off[p], F = off[p + 1] - o0;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * J) return;
  const long long k = i / J;
  const int j = (int)(i - k * J);
  const float* r = pred + ((o0 + k) * J + j) * 3;
  float x = r[0], y = r[1];
  const float z = r[2];
  const long long t = frames[o0 + k];
  const float* kpp = kp + (long long)p * T * J * D;
  if (k > 0) {
    const float* a = kpp + t * J * D;
    const float* b = kpp + frames[o0] * J * D;
    x = __fsub_rn(x, __fdiv_rn(limb_mean(a, b, D, 0), 500.f));
    y = __fadd_rn(y, __fdiv_rn(limb_mean(a, b, D, 1), 500.f));
  }
  if (common_part) {
    int kc = INT_MAX;
    for (int q = 0; q < ncommon_part; ++q) kc = min(kc, common_part[q]);
    if (kc == INT_MAX) {
      x = y = __int_as_float(0x7fc00000);
    } else {
      const long long tc = frames[off[0] + kc];
      const float* a = kp + tc * J * D;                       // person 0
      const float* b = kp + ((long long)T + tc) * J * D;      // person 1
      const float ax = __fdiv_rn(__fdiv_rn(limb_mean(a, b, D, 0), 2.f), 500.f);
      const float ay = __fdiv_rn(__fdiv_rn(limb_mean(a, b, D, 1), 2.f), 500.f);
      x = p == 0 ? __fsub_rn(x, ax) : __fadd_rn(x, ax);
      y = p == 0 ? __fadd_rn(y, ay) : __fsub_rn(y, ay);
    }
  }
  float* w = out + (((long long)p * T + t) * J + j) * 3;
  w[0] = x; w[1] = y; w[2] = z;
}

// pass 1 of z -= amin(z): per block the NaN-propagating minimum of x[3 i + 2], i < n
__global__ void zmin_partial_kernel(const float* __restrict__ x, long long n, float* __restrict__ part) {
  float m = INFINITY;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m = np_minf(x[3 * i + 2], m);
  for (int o = 16; o > 0; o >>= 1) m = np_minf(__shfl_xor_sync(0xffffffffu, m, o), m);
  __shared__ float sh[PREP_BLOCK / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < PREP_BLOCK / 32; ++w) m = np_minf(sh[w], m);
    part[blockIdx.x] = m;
  }
}

// pass 2: every block finishes the minimum from the nb partials in the same order, then x[3 i + 2] -= min
__global__ void zmin_subtract_kernel(float* __restrict__ x, long long n, const float* __restrict__ part, int nb) {
  __shared__ float zmin;
  if (threadIdx.x == 0) {
    float m = part[0];
    for (int q = 1; q < nb; ++q) m = np_minf(part[q], m);
    zmin = m;
  }
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    x[3 * i + 2] = __fsub_rn(x[3 * i + 2], zmin);
}

// revise_skes_real_time (:158-172), one thread per (person, joint): x -= (m_x - cx) / r, y += (m_y - cy) / r with m the
// limb mean of the person's 2D keypoints (J = 17, D floats per keypoint), and the per-block minimum of z
__global__ void revise_rt_kernel(const float* __restrict__ pred, const float* __restrict__ kp, float* __restrict__ out, int M,
                                 int D, float cx, float cy, float r, float* __restrict__ part) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float z = INFINITY;
  if (i < M * 17) {
    const float* a = kp + (long long)(i / 17) * 17 * D;
    const float x = __fsub_rn(pred[3 * i], __fdiv_rn(__fsub_rn(limb_mean(a, nullptr, D, 0), cx), r));
    const float y = __fadd_rn(pred[3 * i + 1], __fdiv_rn(__fsub_rn(limb_mean(a, nullptr, D, 1), cy), r));
    z = pred[3 * i + 2];
    out[3 * i] = x; out[3 * i + 1] = y; out[3 * i + 2] = z;
  }
  for (int o = 16; o > 0; o >>= 1) z = np_minf(__shfl_xor_sync(0xffffffffu, z, o), z);
  __shared__ float sh[PREP_BLOCK / 32];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = z;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 0; w < PREP_BLOCK / 32; ++w) z = np_minf(sh[w], z);
    part[blockIdx.x] = z;
  }
}

// normalize_screen_coordinates (common/camera.py:8-12): X/w*2 - [1, h/w].  numpy evaluates X/w*2 in
// float32 and the subtraction of the Python-float list in float64; the result is rounded to float32
// here (callers cast it: reconstruction.py:143, main.py:46).   image_coordinates (:15-19) is the inverse.
__global__ void screen_norm_kernel(const float* __restrict__ x, float* __restrict__ out, long long n, float w, double hw,
                                   int inverse) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const double c = (idx & 1) ? hw : 1.0;
  if (!inverse) {
    const float s = __fmul_rn(__fdiv_rn(x[idx], w), 2.f);
    out[idx] = (float)((double)s - c);
  } else {
    out[idx] = (float)(((double)x[idx] + c) * (double)w / 2.0);
  }
}

// camera_to_world (common/camera.py:27-28) with one quaternion for every point: qort(q, v) + t
// (common/quaternion.py:4-18: v + 2 * (q0 * (qv x v) + qv x (qv x v)))
__global__ void cam_to_world_kernel(const float* __restrict__ x, float* __restrict__ out, long long npts, float q0, float q1,
                                    float q2, float q3, float t0, float t1, float t2) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npts) return;
  const float vx = x[3 * i], vy = x[3 * i + 1], vz = x[3 * i + 2];
  const float ux = q2 * vz - q3 * vy, uy = q3 * vx - q1 * vz, uz = q1 * vy - q2 * vx;
  const float wx = q2 * uz - q3 * uy, wy = q3 * ux - q1 * uz, wz = q1 * uy - q2 * ux;
  out[3 * i] = vx + 2.f * (q0 * ux + wx) + t0;
  out[3 * i + 1] = vy + 2.f * (q0 * uy + wy) + t1;
  out[3 * i + 2] = vz + 2.f * (q0 * uz + wz) + t2;
}

// ------------------------------------------------------------------------------------------
// N2: mpjpe (common/loss.py:5-11) forward + backward in one pass.  loss = mean_i ||p_i - t_i||;
// d loss / d p_i = (p_i - t_i) / (||.|| n)  (0 where the norm is 0, like torch.norm's backward).
// ------------------------------------------------------------------------------------------
constexpr int MPJPE_BLOCKS = 256;

__global__ void mpjpe_kernel(const float* __restrict__ pred, const float* __restrict__ tgt, long long n, int D,
                             float gscale, float* __restrict__ dpred, double* __restrict__ partial) {
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float d[4], s = 0.f;
    for (int c = 0; c < D; ++c) { d[c] = pred[i * D + c] - tgt[i * D + c]; s = fmaf(d[c], d[c], s); }
    const float nrm = sqrtf(s);
    acc += (double)nrm;
    if (dpred) {
      const float k = nrm > 0.f ? gscale / nrm : 0.f;
      for (int c = 0; c < D; ++c) dpred[i * D + c] = d[c] * k;
    }
  }
  __shared__ double sh[32];
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) partial[blockIdx.x] = v;
  }
}

__global__ void mpjpe_final_kernel(const double* __restrict__ partial, int nb, long long n, float* __restrict__ loss) {
  double v = 0.0;
  for (int i = threadIdx.x; i < nb; i += 32) v += partial[i];
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (threadIdx.x == 0) *loss = (float)(v / (double)n);
}

// ------------------------------------------------------------------------------------------
// N2: p_mpjpe (common/loss.py:14-53): per frame, similarity-Procrustes alignment of the prediction to
// the target (3x3 SVD), then the mean joint distance.  One warp per frame, lanes over joints; the 3x3
// decomposition runs in double (Jacobi on H^T H) on every lane redundantly.  R is a proper rotation for every rank of
// H (planar and collinear frames included); a frame with zero spread divides by a zero norm and gives NaN, as the
// reference does.
// ------------------------------------------------------------------------------------------
constexpr double PM_NOISE = 1e-12;                        // |H v| below PM_NOISE s0 is rounding noise, not a direction

__device__ __forceinline__ double warp_sum_d(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ inline void jacobi_eig3(double a[3][3], double v[3][3]) {   // a symmetric -> a diagonal, v eigenvectors (columns)
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) v[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 12; ++sweep) {
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = a[p][q];
        if (fabs(apq) < 1e-300) continue;
        const double th = (a[q][q] - a[p][p]) / (2.0 * apq);
        const double tt = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
        for (int k = 0; k < 3; ++k) {
          const double akp = a[k][p], akq = a[k][q];
          a[k][p] = c * akp - s * akq; a[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 3; ++k) {
          const double apk = a[p][k], aqk = a[q][k];
          a[p][k] = c * apk - s * aqk; a[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 3; ++k) {
          const double vkp = v[k][p], vkq = v[k][q];
          v[k][p] = c * vkp - s * vkq; v[k][q] = s * vkp + c * vkq;
        }
      }
  }
}

__global__ void p_mpjpe_kernel(const float* __restrict__ pred, const float* __restrict__ tgt, float* __restrict__ err,
                               int N, int J) {
  const int frame = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (frame >= N) return;
  const bool on = lane < J;
  double X[3] = {0, 0, 0}, Y[3] = {0, 0, 0};
  if (on)
    for (int c = 0; c < 3; ++c) { X[c] = tgt[((long long)frame * J + lane) * 3 + c]; Y[c] = pred[((long long)frame * J + lane) * 3 + c]; }
  double muX[3], muY[3];
  for (int c = 0; c < 3; ++c) { muX[c] = warp_sum_d(X[c]) / J; muY[c] = warp_sum_d(Y[c]) / J; }
  double X0[3], Y0[3], nx = 0, ny = 0;
  for (int c = 0; c < 3; ++c) {
    X0[c] = on ? X[c] - muX[c] : 0.0; Y0[c] = on ? Y[c] - muY[c] : 0.0;
    nx += X0[c] * X0[c]; ny += Y0[c] * Y0[c];
  }
  const double normX = sqrt(warp_sum_d(nx)), normY = sqrt(warp_sum_d(ny));
  for (int c = 0; c < 3; ++c) { X0[c] /= normX; Y0[c] /= normY; }
  double H[3][3];                                         // H = X0^T Y0   (:33)
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) H[i][j] = warp_sum_d(X0[i] * Y0[j]);
  // SVD  H = U diag(s) V^T  from the eigen-decomposition of H^T H
  double B[3][3], V[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) B[i][j] = H[0][i] * H[0][j] + H[1][i] * H[1][j] + H[2][i] * H[2][j];
  jacobi_eig3(B, V);
  double lam[3] = {B[0][0], B[1][1], B[2][2]};
  int ord[3] = {0, 1, 2};                                 // descending eigenvalues (numpy's singular-value order)
  for (int i = 0; i < 2; ++i) for (int j = 0; j < 2 - i; ++j)
    if (lam[ord[j]] < lam[ord[j + 1]]) { int tq = ord[j]; ord[j] = ord[j + 1]; ord[j + 1] = tq; }
  double Vs[3][3], U[3][3], s[3], w[3][3];                // w[:,k] = H v_k
  for (int k = 0; k < 3; ++k)
    for (int i = 0; i < 3; ++i) Vs[i][k] = V[i][ord[k]];
  for (int k = 0; k < 3; ++k)
    for (int i = 0; i < 3; ++i) w[i][k] = H[i][0] * Vs[0][k] + H[i][1] * Vs[1][k] + H[i][2] * Vs[2][k];
  // U from H v_k by Gram-Schmidt, orthonormal at every rank of H.  sqrt(lambda_k) cannot be the divisor: H^T H carries
  // rounding of ~1e-16 s0^2, so for a planar or collinear frame the "zero" singular values come out near 1e-8 s0 and
  // H v_k / sqrt(lambda_k) is noise of no particular length.  s_k = u_k^T H v_k.
  const double n0 = sqrt(w[0][0] * w[0][0] + w[1][0] * w[1][0] + w[2][0] * w[2][0]);
  for (int i = 0; i < 3; ++i) U[i][0] = n0 > 0.0 ? w[i][0] / n0 : (i == 0 ? 1.0 : 0.0);
  double u1[3] = {w[0][1], w[1][1], w[2][1]};
  for (int pass = 0; pass < 2; ++pass) {                  // twice: orthogonal to rounding even when H v1 is mostly u0
    const double p = U[0][0] * u1[0] + U[1][0] * u1[1] + U[2][0] * u1[2];
    for (int i = 0; i < 3; ++i) u1[i] -= p * U[i][0];
  }
  const double n1 = sqrt(u1[0] * u1[0] + u1[1] * u1[1] + u1[2] * u1[2]);
  if (n1 > PM_NOISE * n0) {
    for (int i = 0; i < 3; ++i) U[i][1] = u1[i] / n1;
  } else {                                                // rank(H) <= 1: any unit vector orthogonal to u0 (u0 x e_m,
    int m = 0;                                            // e_m the axis of u0's smallest component)
    for (int i = 1; i < 3; ++i) if (fabs(U[i][0]) < fabs(U[m][0])) m = i;
    const double e[3] = {m == 0 ? 1.0 : 0.0, m == 1 ? 1.0 : 0.0, m == 2 ? 1.0 : 0.0};
    const double c[3] = {U[1][0] * e[2] - U[2][0] * e[1], U[2][0] * e[0] - U[0][0] * e[2], U[0][0] * e[1] - U[1][0] * e[0]};
    const double nc = sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
    for (int i = 0; i < 3; ++i) U[i][1] = c[i] / nc;
  }
  {                                                       // u2 = +-(u0 x u1), the sign of (H v2).(u0 x u1); + at noise
    const double c[3] = {U[1][0] * U[2][1] - U[2][0] * U[1][1], U[2][0] * U[0][1] - U[0][0] * U[2][1],
                         U[0][0] * U[1][1] - U[1][0] * U[0][1]};
    const double d = w[0][2] * c[0] + w[1][2] * c[1] + w[2][2] * c[2];
    const double sg = (d < 0.0 && -d > PM_NOISE * n0) ? -1.0 : 1.0;
    for (int i = 0; i < 3; ++i) U[i][2] = sg * c[i];
    s[0] = n0;
    s[1] = U[0][1] * w[0][1] + U[1][1] * w[1][1] + U[2][1] * w[2][1];
    s[2] = sg * d;
  }
  auto det3 = [](double m[3][3]) {
    return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
           m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
  };
  if (det3(Vs) * det3(U) < 0.0) {                         // det(R) = -1: flip the last singular direction (:39-43)
    for (int i = 0; i < 3; ++i) Vs[i][2] = -Vs[i][2];
    s[2] = -s[2];
  }
  double R[3][3];                                         // R = V U^T
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R[i][j] = Vs[i][0] * U[j][0] + Vs[i][1] * U[j][1] + Vs[i][2] * U[j][2];
  const double a = (s[0] + s[1] + s[2]) * normX / normY;  // scale (:45-47)
  double e = 0.0;
  if (on) {
    double d2 = 0.0;
    for (int c = 0; c < 3; ++c) {
      const double yr = Y[0] * R[0][c] + Y[1] * R[1][c] + Y[2] * R[2][c];
      const double mr = muY[0] * R[0][c] + muY[1] * R[1][c] + muY[2] * R[2][c];
      const double al = a * yr + (muX[c] - a * mr);       // a * pred . R + t   (:48-51)
      d2 += (al - X[c]) * (al - X[c]);
    }
    e = sqrt(d2);
  }
  e = warp_sum_d(e);
  if (lane == 0) err[frame] = (float)(e / J);
}

// ------------------------------------------------------------------------------------------
// N2: Adam with amsgrad (trainval.py:78 optim.Adam(..., amsgrad=True); torch/optim/adam.py single-tensor
// update) over every parameter in ONE launch.  table[i] = {param ptr, grad ptr, state offset, count}:
// a chunk of <= ADAM_CHUNK elements of one tensor; the moments live in flat state buffers.
// ------------------------------------------------------------------------------------------
constexpr int ADAM_CHUNK = 4096;

__global__ void adam_multi_kernel(const long long* __restrict__ table, float* __restrict__ exp_avg,
                                  float* __restrict__ exp_avg_sq, float* __restrict__ max_sq, float one_m_b1, float b2,
                                  float one_m_b2, float step_size, float bc2_sqrt, float eps, float wd) {
  const long long* e = table + 4LL * blockIdx.x;
  float* p = reinterpret_cast<float*>(e[0]);
  const float* g = reinterpret_cast<const float*>(e[1]);
  const long long so = e[2];
  const int cnt = (int)e[3];
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
    float pv = p[i], gv = g[i];
    if (wd != 0.f) gv = fmaf(wd, pv, gv);
    float m = exp_avg[so + i], v = exp_avg_sq[so + i];
    m = m + one_m_b1 * (gv - m);                          // exp_avg.lerp_(grad, 1 - beta1)
    v = v * b2 + one_m_b2 * gv * gv;                      // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    exp_avg[so + i] = m;
    exp_avg_sq[so + i] = v;
    float vd = v;
    if (max_sq) { vd = fmaxf(max_sq[so + i], v); max_sq[so + i] = vd; }
    const float denom = sqrtf(vd) / bc2_sqrt + eps;
    p[i] = pv - step_size * (m / denom);
  }
}

}  // namespace gast

extern "C" int gast_chunk_gather(const float* poses_2d, const float* poses_3d, const float* cameras,
                                 const int64_t* seq_start, int32_t n_seq, const int32_t* pairs, int32_t B,
                                 int32_t chunk, int32_t pad, int32_t causal_shift, int32_t J2, int32_t F2, int32_t J3,
                                 int32_t ncam, int32_t n_sym2, const int32_t* kps_left, const int32_t* kps_right,
                                 int32_t n_sym3, const int32_t* joints_left, const int32_t* joints_right,
                                 float* batch_2d, float* batch_3d, float* batch_cam, void* stream) {
  if (!poses_2d || !seq_start || !pairs || !batch_2d || B <= 0 || chunk <= 0 || pad < 0 || n_seq <= 0 || J2 <= 0 || F2 <= 0)
    return fail("gast_chunk_gather: bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  JointPerm p2, p3;
  if (make_perm(J2, n_sym2, kps_left, kps_right, &p2)) return 1;
  const int Tc = chunk + 2 * pad;
  const long long n2 = (long long)B * Tc * J2 * F2;
  chunk_gather_kernel<<<cdiv(n2, 256), 256, 0, st>>>(poses_2d, reinterpret_cast<const long long*>(seq_start), pairs,
                                                     batch_2d, B, Tc, J2, F2, pad + causal_shift, p2);
  if (poses_3d && batch_3d) {
    if (make_perm(J3, n_sym3, joints_left, joints_right, &p3)) return 1;
    const long long n3 = (long long)B * chunk * J3 * 3;
    chunk_gather_kernel<<<cdiv(n3, 256), 256, 0, st>>>(poses_3d, reinterpret_cast<const long long*>(seq_start), pairs,
                                                       batch_3d, B, chunk, J3, 3, 0, p3);
  }
  if (cameras && batch_cam && ncam > 0)
    chunk_cam_kernel<<<cdiv((long long)B * ncam, 256), 256, 0, st>>>(cameras, pairs, batch_cam, B, ncam);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_keypoints_convert(const float* kpts, float* out, int32_t* valid, int32_t T, int32_t J_in, int32_t mode,
                                      void* stream) {
  if (!kpts || !out || T <= 0) return fail("gast_keypoints_convert: bad arguments");
  if ((mode == 0 && J_in != 17) || (mode == 1 && J_in != 16) || (mode == 2 && J_in < 22) || mode < 0 || mode > 2)
    return fail("gast_keypoints_convert: mode %d does not take %d joints", mode, J_in);
  kpt_convert_kernel<<<cdiv(T, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(kpts, out, valid, T, J_in, mode);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_normalize_screen(const float* x, float* out, int64_t n_points, float w, float h, int32_t inverse,
                                     void* stream) {
  if (!x || !out || n_points <= 0 || w == 0.f) return fail("gast_normalize_screen: bad arguments");
  const long long n = 2 * n_points;
  screen_norm_kernel<<<cdiv(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, out, n, w, (double)h / (double)w,
                                                                                      inverse);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_camera_to_world(const float* x, float* out, int64_t n_points, const float* q, const float* t,
                                    void* stream) {
  if (!x || !out || !q || n_points <= 0) return fail("gast_camera_to_world: bad arguments");
  cam_to_world_kernel<<<cdiv(n_points, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, out, n_points, q[0], q[1], q[2], q[3], t ? t[0] : 0.f, t ? t[1] : 0.f, t ? t[2] : 0.f);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" size_t gast_mpjpe_workspace_bytes(void) { return sizeof(double) * MPJPE_BLOCKS; }

extern "C" int gast_mpjpe(const float* pred, const float* target, int64_t n_points, int32_t D, float* loss, float* dpred,
                          float grad_scale, void* workspace, void* stream) {
  if (!pred || !target || !loss || !workspace || n_points <= 0 || D < 1 || D > 4) return fail("gast_mpjpe: bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nb = (int)std::min<long long>(MPJPE_BLOCKS, (n_points + 255) / 256);
  mpjpe_kernel<<<nb, 256, 0, st>>>(pred, target, n_points, D, grad_scale / (float)n_points, dpred,
                                  reinterpret_cast<double*>(workspace));
  mpjpe_final_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const double*>(workspace), nb, n_points, loss);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_p_mpjpe(const float* pred, const float* target, int32_t N, int32_t J, float* per_frame, void* stream) {
  if (!pred || !target || !per_frame || N <= 0 || J < 3 || J > 32) return fail("gast_p_mpjpe: bad arguments (3 <= J <= 32)");
  p_mpjpe_kernel<<<cdiv((long long)N * 32, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pred, target, per_frame, N, J);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int32_t gast_adam_chunk(void) { return ADAM_CHUNK; }

extern "C" int gast_adam_step(const int64_t* table, int32_t n_chunks, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                              double lr, double beta1, double beta2, double eps, double weight_decay, int64_t step,
                              void* stream) {
  if (!table || !exp_avg || !exp_avg_sq || n_chunks <= 0 || step < 1) return fail("gast_adam_step: bad arguments");
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  adam_multi_kernel<<<n_chunks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(table), exp_avg, exp_avg_sq, max_exp_avg_sq, (float)(1.0 - beta1), (float)beta2,
      (float)(1.0 - beta2), (float)(lr / bc1), (float)sqrt(bc2), (float)eps, (float)weight_decay);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_h36m_coco_format(const float* kpts, const float* scores, int32_t P, int32_t T, float* out_kpts,
                                     float* out_scores, int32_t* valid, int32_t* keep, void* stream) {
  if (!kpts || !scores || !out_kpts || !out_scores || !valid || !keep || P <= 0 || T <= 0)
    return fail("gast_h36m_coco_format: bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUDA_OK(cudaMemsetAsync(keep, 0, sizeof(int32_t) * P, st));
  h36m_coco_format_kernel<<<cdiv((long long)P * T, 128), 128, 0, st>>>(kpts, scores, out_kpts, out_scores, valid, keep, P, T);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_revise_kpts(const float* kpts, const float* scores, const int32_t* valid, int32_t P, int32_t T, int32_t J,
                                float* out, void* stream) {
  if (!kpts || !scores || !valid || !out || P <= 0 || T <= 0 || J < 7) return fail("gast_revise_kpts: bad arguments (J >= 7)");
  const long long PT = (long long)P * T;
  revise_kpts_kernel<<<cdiv(PT, 128), 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(kpts, scores, valid, out, PT, J);
  CUDA_OK(cudaGetLastError());
  return 0;
}

namespace gast {
constexpr int PREP_COMMON_BLOCKS = 64, PREP_ZMIN_BLOCKS = 512;
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
}  // namespace gast

extern "C" size_t gast_revise_skes_workspace_bytes(int32_t P, int32_t T) {
  if (P <= 0 || T <= 0) return 0;
  return align256(sizeof(int64_t) * (P + 1)) + align256(sizeof(int32_t) * (size_t)T) +
         align256(sizeof(int32_t) * PREP_COMMON_BLOCKS) + align256(sizeof(float) * PREP_ZMIN_BLOCKS);
}

extern "C" int gast_revise_skes(const float* pred, const int64_t* frames, const int64_t* offsets, int32_t P, int32_t T,
                                int32_t J, int32_t D, const float* kpts, float* out, void* workspace, size_t workspace_bytes,
                                void* stream) {
  if (!pred || !frames || !offsets || !kpts || !out || !workspace || P <= 0 || T <= 0 || J < 15 || D < 2)
    return fail("gast_revise_skes: bad arguments (J >= 15, D >= 2)");
  if (workspace_bytes < gast_revise_skes_workspace_bytes(P, T))
    return fail("gast_revise_skes: workspace of %zu bytes, %zu needed", workspace_bytes, gast_revise_skes_workspace_bytes(P, T));
  long long maxF = 0;
  for (int p = 0; p < P; ++p) {
    const long long F = offsets[p + 1] - offsets[p];
    if (offsets[0] != 0 || F < 0 || F > T) return fail("gast_revise_skes: person %d has %lld frames, T = %d", p, F, T);
    maxF = std::max(maxF, F);
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  char* ws = reinterpret_cast<char*>(workspace);
  long long* doff = reinterpret_cast<long long*>(ws);
  ws += align256(sizeof(int64_t) * (P + 1));
  int* mask1 = reinterpret_cast<int*>(ws);
  ws += align256(sizeof(int32_t) * (size_t)T);
  int* cpart = reinterpret_cast<int*>(ws);
  ws += align256(sizeof(int32_t) * PREP_COMMON_BLOCKS);
  float* zpart = reinterpret_cast<float*>(ws);
  CUDA_OK(cudaMemcpyAsync(doff, offsets, sizeof(int64_t) * (P + 1), cudaMemcpyHostToDevice, st));
  CUDA_OK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)P * T * J * 3, st));
  const long long* fr = reinterpret_cast<const long long*>(frames);
  const int* common = nullptr;
  int ncommon = 0;
  if (P == 2) {                                           // preprocess.py:138-141
    const long long F0 = offsets[1], F1 = offsets[2] - offsets[1];
    CUDA_OK(cudaMemsetAsync(mask1, 0, sizeof(int32_t) * (size_t)T, st));
    if (F1 > 0) mask_scatter_kernel<<<cdiv(F1, 256), 256, 0, st>>>(fr + F0, (int)F1, mask1);
    ncommon = (int)std::max<long long>(1, std::min<long long>(PREP_COMMON_BLOCKS, cdiv(F0, PREP_BLOCK)));
    first_common_kernel<<<ncommon, PREP_BLOCK, 0, st>>>(fr, (int)F0, mask1, cpart);
    common = cpart;
  }
  if (maxF > 0) {
    dim3 grid(cdiv(maxF * J, 128), P);
    revise_skes_kernel<<<grid, 128, 0, st>>>(pred, fr, doff, kpts, out, T, J, D, common, ncommon);
  }
  const long long n = (long long)P * T * J;                // preprocess.py:153, over the whole output
  const int nb = (int)std::min<long long>(PREP_ZMIN_BLOCKS, cdiv(n, PREP_BLOCK));
  zmin_partial_kernel<<<nb, PREP_BLOCK, 0, st>>>(out, n, zpart);
  zmin_subtract_kernel<<<nb, PREP_BLOCK, 0, st>>>(out, n, zpart, nb);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" size_t gast_revise_skes_real_time_workspace_bytes(int32_t M) {
  return M > 0 ? sizeof(float) * cdiv((long long)M * 17, PREP_BLOCK) : 0;
}

extern "C" int gast_revise_skes_real_time(const float* pred, const float* kpts, int32_t M, int32_t J, int32_t D, double width,
                                          float* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (J != 17) return fail("gast_revise_skes_real_time: the reference places 17 joints, got %d", J);
  if (!pred || !kpts || !out || !workspace || M <= 0 || D < 2) return fail("gast_revise_skes_real_time: bad arguments");
  if (workspace_bytes < gast_revise_skes_real_time_workspace_bytes(M))
    return fail("gast_revise_skes_real_time: workspace of %zu bytes, %zu needed", workspace_bytes,
                gast_revise_skes_real_time_workspace_bytes(M));
  // preprocess.py:159,167-168 under NumPy 2's promotion: the Python-float constants are rounded to float32 and every
  // operation is float32
  const float cx = (float)(3.0 * width / 5.0), cy = (float)(width / 5.0), r = (float)(500.0 * (width / 1920.0));
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int nb = (int)cdiv((long long)M * 17, PREP_BLOCK);
  float* part = reinterpret_cast<float*>(workspace);
  revise_rt_kernel<<<nb, PREP_BLOCK, 0, st>>>(pred, kpts, out, M, D, cx, cy, r, part);
  zmin_subtract_kernel<<<nb, PREP_BLOCK, 0, st>>>(out, (long long)M * 17, part, nb);
  CUDA_OK(cudaGetLastError());
  return 0;
}
