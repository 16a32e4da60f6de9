// Shared device-side types of libgast_b200 (sm_90a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace gast {

constexpr float BN_EPS = 1e-5f;  // nn.BatchNorm2d default used throughout the reference

// Frame remap of a gathered operand: output frame f = b*T_out + t  ->  input frame
// b*T_in + t*t_mul + t_off.  Identity is {1,1,1,0} on flattened frames.
struct RowMap {
  int T_out, T_in, t_mul, t_off;
};

__host__ __device__ inline long long map_frame(const RowMap& m, long long f) {
  long long b = f / m.T_out;
  long long t = f - b * m.T_out;
  return b * m.T_in + t * m.t_mul + m.t_off;
}

// One K-segment of the A operand: rows gathered from `base` (channels-last, row stride ld).
// K may span several temporal taps: k -> (tap = k / Kc, c = k % Kc), the tap adds
// tap * tap_stride floats (dilation * J * ld) to the row address.
struct ASeg {
  const float* base;
  int ld;
  int K;
  int Kc;
  long long tap_stride;
  RowMap map;
};

// Sparse row structure of a LocalGraph mask (J <= 32, nnz <= 160), row-major nonzero order
// == the order of the learnable `e` (local_attention.py:25,41).
struct NbrTable {
  unsigned char row_ptr[36];
  unsigned char col[164];
};

struct GemmP {
  ASeg seg[3];
  int nseg;
  const float* W;   // [N][ldw], K-major
  int ldw;
  int N;
  int F;            // output frames
  int J;
  int fpt;          // frames per 128-row tile
  float* out;
  int ld_out;
  const float* bias;
  int relu;
  const float* res; // optional residual, added after the activation (gast_net.py:174)
  int res_ld;
  RowMap res_map;
  // EPI_SEMCH
  const float* coef[2];   // [nnz][C], softmaxed adjacency x BN scale
  const float* shift;     // [2][C] BN shift (or SemGraphConv bias), may be null
  int C;
  int tiles_per_mask;
  NbrTable nbr[2];
  // EPI_GLOBAL
  const float* ab;  // [rows][2*heads]: a_h(i), b_h(j)
  const float* ck;  // [heads][J][J]
  const float* bg;  // [N]
  int heads;
  int Cg;
};

__device__ __forceinline__ float4 ldg4(const float* p) {
  return __ldg(reinterpret_cast<const float4*>(p));
}

// Element access of the HBM-side kernels, which are templated on the activation type (float, or __half under
// gast_set_activation_dtype(h, GAST_F16)): loads widen to fp32 and stores round to nearest, arithmetic stays fp32.
__device__ __forceinline__ float ld1(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ld1(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float4 ld4(const float* p) { return ldg4(p); }
__device__ __forceinline__ float4 ld4(const __half* p) {   // 4 halves, 8-byte aligned
  const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void st1(float* p, float v) { *p = v; }
__device__ __forceinline__ void st1(__half* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void st4(__half* p, float4 v) {
  const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&a);
  u.y = *reinterpret_cast<const uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace gast
