// The box geometry between SORT's tracks and the 2D pose net (lib/pose/hrnet/lib/utils/utilitys.py:107-170,
// lib/pose/hrnet/lib/utils/transforms.py:57-89), shared by the offline crop records (records.cuh) and the live tick's
// slots (live.cuh): which rows a frame's track count selects, box_to_center_scale, get_affine_transform's float32
// triangles and cv2.getAffineTransform's 6 x 6 LU.
//
// The matrices are cv2.getAffineTransform's: OpenCV builds a 6 x 6 system and solves it with LUImpl (partial
// pivoting, d = -1 / A[i][i], row updates A[j][k] += alpha * A[i][k], back-substitution with k ascending, b[i] = s /
// A[i][i]), all of it plain unfused double in its x86 build.  Every step here is an explicit round-to-nearest
// intrinsic in that order (nvcc would otherwise contract a * b + c into an FMA), and so are the float32 / float64
// steps of the box geometry before it, so the results equal the host functions bit for bit (DESIGN.md §8.9).
#pragma once
#include <math.h>

namespace gast {

// status bits above SORT's own word (include/gast_b200.h)
constexpr int REC_ST_TRACKS = 0x100, REC_ST_NONFINITE = 0x200, REC_ST_EMPTY = 0x400, REC_ST_MATRIX = 0x800;
constexpr int REC_ST_FRAME = REC_ST_TRACKS | REC_ST_NONFINITE | REC_ST_EMPTY;   // bits that name a frame

// the boxes a frame of k tracks gives (select_tracks, gen_img_kpts:146-150): none for k <= 0, the lone track for
// k = 1, else the last num_person rows; -1 for a count the host path refuses (2 <= k < num_person) or that cannot be
// SORT's
__device__ __forceinline__ int rec_count(int k, int num_person, int cap) {
  if (k < -1 || k > cap) return -1;
  if (k <= 0) return 0;
  if (k == 1) return 1;
  return k >= num_person ? num_person : -1;
}

// box_to_center_scale of the corners (x1, y1, x2, y2) with aspect = H / W (PreProcess passes the frame's (H, W) in the
// model-size slots): the float32 center (c0, c1) and scale (s0, s1); bits gets REC_ST_NONFINITE for a non-finite
// corner, else REC_ST_EMPTY for a non-positive width and height
__device__ __forceinline__ void rec_center_scale(double x1, double y1, double x2, double y2, double aspect, int& bits,
                                                 float& c0, float& c1, float& s0, float& s1) {
  double bw = __dsub_rn(x2, x1), bh = __dsub_rn(y2, y1);
  if (!(isfinite(x1) && isfinite(y1) && isfinite(x2) && isfinite(y2)))
    bits |= REC_ST_NONFINITE;
  else if (bw <= 0.0 && bh <= 0.0)
    bits |= REC_ST_EMPTY;
  c0 = __double2float_rn(__dadd_rn(x1, __dmul_rn(bw, 0.5)));
  c1 = __double2float_rn(__dadd_rn(y1, __dmul_rn(bh, 0.5)));
  if (bw > __dmul_rn(aspect, bh))
    bh = __ddiv_rn(bw, aspect);
  else if (bw < __dmul_rn(aspect, bh))
    bw = __dmul_rn(bh, aspect);
  s0 = __double2float_rn(__ddiv_rn(bw, 200.0));
  s1 = __double2float_rn(__ddiv_rn(bh, 200.0));
  if (c0 != -1.f) {
    s0 = __fmul_rn(s0, 1.25f);
    s1 = __fmul_rn(s1, 1.25f);
  }
}

// get_affine_transform's float32 triangles (rot 0, no shift) for an output of ow x oh: src[6] in the frame around
// the box, dst[6] in the output, as (x, y) pairs
__device__ __forceinline__ void rec_triangles(float c0, float c1, float s0, int ow, int oh, float (&src)[6],
                                              float (&dst)[6]) {
  const float src_w = __fmul_rn(s0, 200.f);
  src[0] = c0;
  src[1] = c1;
  // get_dir's result is float64: center + (0, src_w * -0.5) in double, stored into float32
  src[2] = __double2float_rn(__dadd_rn((double)c0, 0.0));
  src[3] = __double2float_rn(__dadd_rn((double)c1, (double)__fmul_rn(src_w, -0.5f)));
  const double hw = __dmul_rn((double)ow, 0.5), hh = __dmul_rn((double)oh, 0.5);
  dst[0] = __double2float_rn(hw);
  dst[1] = __double2float_rn(hh);
  dst[2] = __double2float_rn(__dadd_rn(hw, 0.0));
  dst[3] = __double2float_rn(__dadd_rn(hh, (double)__double2float_rn(__dmul_rn((double)ow, -0.5))));
  // get_3rd_point in float32: b + (-(a - b).y, (a - b).x)
  const float sd0 = __fsub_rn(src[0], src[2]), sd1 = __fsub_rn(src[1], src[3]);
  src[4] = __fadd_rn(src[2], -sd1);
  src[5] = __fadd_rn(src[3], sd0);
  const float dd0 = __fsub_rn(dst[0], dst[2]), dd1 = __fsub_rn(dst[1], dst[3]);
  dst[4] = __fadd_rn(dst[2], -dd1);
  dst[5] = __fadd_rn(dst[3], dd0);
}

// cv2.getAffineTransform(src, dst): the 6 x 6 system and LUImpl; a pivot below 100 * DBL_EPSILON makes solve()
// fail and the matrix all zero, as OpenCV returns it
__device__ __forceinline__ void rec_affine(const float (&src)[6], const float (&dst)[6], double (&m)[6]) {
  double a[6][6], b[6];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double x = src[2 * i], y = src[2 * i + 1];
    a[2 * i][0] = x;   a[2 * i][1] = y;   a[2 * i][2] = 1.0;
    a[2 * i][3] = 0.0; a[2 * i][4] = 0.0; a[2 * i][5] = 0.0;
    a[2 * i + 1][0] = 0.0; a[2 * i + 1][1] = 0.0; a[2 * i + 1][2] = 0.0;
    a[2 * i + 1][3] = x;   a[2 * i + 1][4] = y;   a[2 * i + 1][5] = 1.0;
    b[2 * i] = dst[2 * i];
    b[2 * i + 1] = dst[2 * i + 1];
  }
  bool singular = false;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    int k = i;
    double best = fabs(a[i][i]);
#pragma unroll
    for (int j = i + 1; j < 6; ++j)
      if (fabs(a[j][i]) > best) {
        best = fabs(a[j][i]);
        k = j;
      }
    singular |= best < 100.0 * 2.220446049250313e-16;
#pragma unroll
    for (int j = i + 1; j < 6; ++j)
      if (k == j) {
#pragma unroll
        for (int c = i; c < 6; ++c) {
          const double t = a[i][c];
          a[i][c] = a[j][c];
          a[j][c] = t;
        }
        const double t = b[i];
        b[i] = b[j];
        b[j] = t;
      }
    const double d = __ddiv_rn(-1.0, a[i][i]);
#pragma unroll
    for (int j = i + 1; j < 6; ++j) {
      const double alpha = __dmul_rn(a[j][i], d);
#pragma unroll
      for (int c = i + 1; c < 6; ++c) a[j][c] = __dadd_rn(a[j][c], __dmul_rn(alpha, a[i][c]));
      b[j] = __dadd_rn(b[j], __dmul_rn(alpha, b[i]));
    }
  }
#pragma unroll
  for (int i = 5; i >= 0; --i) {
    double s = b[i];
#pragma unroll
    for (int c = i + 1; c < 6; ++c) s = __dsub_rn(s, __dmul_rn(a[i][c], b[c]));
    b[i] = __ddiv_rn(s, a[i][i]);
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) m[i] = singular ? 0.0 : b[i];
}

}  // namespace gast
