// The reconstruction's animation frames (tools/vis_h36m.py:58-249, tools/visualization.py:84-227), rasterised on
// the device: one uint8 RGB frame per time step, an input panel (the video frame with the 2D skeleton and joint
// discs) followed by the 3D panels (the lifted skeletons under the reference's view), each S x S pixels.
//
// One thread owns one output pixel and writes it once; a block first stages its frame's projected joints in shared
// memory.  There are no atomics and no sums across threads, so a pixel depends only on its own frame's inputs and
// the call's geometry: every call repeats bit for bit, and a frame renders the same in any frame range.  Every
// float operation is an explicit round-to-nearest intrinsic (no FMA contraction), in the order DESIGN.md §8.5 writes
// down, so tests/renderref.py restates the kernel in numpy float32 exactly.
//
// Included at the end of gast_api.cu (uses fail / CUDA_OK / cdiv).
#pragma once
#include <math.h>

namespace gast {

constexpr int RENDER_MAX_J = 32;        // joints per skeleton (bit masks and the parents table)
constexpr int RENDER_MAX_PTS = 256;     // staged points per panel: persons x J (input), poses x J (shared 3D panel)
constexpr int RENDER_MAX_PANELS = 8;    // 3D panels
constexpr int RENDER_TILE = 16;         // a block renders a 16 x 16 pixel tile of one panel of one frame

// Everything but the per-frame data, passed by value.  geo[] is gast_render_geometry's output.
struct RenderParams {
  int M, J, n_pose, n_panel, shared, follow_root, bones_2d, n_bones, S, Hin, Win;
  long long kp_frame, pose_stride, video_frame;   // floats per keypoint frame, floats per pose entry, bytes per frame
  int parents[RENDER_MAX_J];
  unsigned char color[RENDER_MAX_J][3];
  unsigned right_mask;
  float geo[20];
};

__device__ __forceinline__ float rfa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float rfs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float rfm(float a, float b) { return __fmul_rn(a, b); }

// distance from the pixel centre w = (X, Y) - A to the segment A -> A + d, and the segment parameter of the nearest
// point (0 at A, 1 at B)
__device__ __forceinline__ float seg_dist(float wx, float wy, float dx, float dy, float* t_out) {
  const float l2 = rfa(rfm(dx, dx), rfm(dy, dy));
  float t = 0.f;
  if (l2 > 0.f) t = fminf(fmaxf(__fdiv_rn(rfa(rfm(wx, dx), rfm(wy, dy)), l2), 0.f), 1.f);
  const float ex = rfs(wx, rfm(t, dx)), ey = rfs(wy, rfm(t, dy));
  *t_out = t;
  return __fsqrt_rn(rfa(rfm(ex, ex), rfm(ey, ey)));
}

__device__ __forceinline__ float lerp_rn(float c, float target, float cov) { return rfa(c, rfm(cov, rfs(target, c))); }

__global__ void __launch_bounds__(RENDER_TILE * RENDER_TILE)
render_kernel(const float* __restrict__ kp, const float* __restrict__ poses, const unsigned char* __restrict__ video,
              const RenderParams p, long long f_first, unsigned char* __restrict__ out) {
  __shared__ float4 pts[RENDER_MAX_PTS];
  const int tiles_x = (p.S + RENDER_TILE - 1) / RENDER_TILE;
  const int panel = blockIdx.y;
  const long long f = (long long)blockIdx.z, g = f_first + f;        // f: output frame of this launch, g: source frame
  const int tid = threadIdx.y * RENDER_TILE + threadIdx.x;
  const float* geo = p.geo;
  const float half = geo[19];

  // stage the panel's points: panel pixel coordinates (X, Y) and, for the 3D panels, the depth dz
  int n_pts, e_count;
  if (panel == 0) {
    e_count = p.M;
    n_pts = p.M * p.J;
    const float* k = kp + g * p.kp_frame;
    for (int i = tid; i < n_pts; i += RENDER_TILE * RENDER_TILE) {
      const float X = rfa(geo[13], rfm(rfa(k[2 * i], 0.5f), geo[12]));
      const float Y = rfa(geo[14], rfm(rfa(k[2 * i + 1], 0.5f), geo[12]));
      pts[i] = make_float4(X, Y, 0.f, 0.f);
    }
  } else {
    const int e0 = p.shared ? 0 : panel - 1;
    e_count = p.shared ? p.n_pose : 1;
    n_pts = e_count * p.J;
    for (int i = tid; i < n_pts; i += RENDER_TILE * RENDER_TILE) {
      const int e = e0 + i / p.J, j = i - (i / p.J) * p.J;
      const float* fr = poses + e * p.pose_stride + g * p.J * 3;
      float q0 = fr[3 * j], q1 = fr[3 * j + 1];
      const float q2 = fr[3 * j + 2];
      if (p.follow_root) {
        q0 = rfs(q0, fr[0]);
        q1 = rfs(q1, fr[1]);
      }
      const float sx = rfa(rfa(rfa(rfm(geo[0], q0), rfm(geo[1], q1)), rfm(geo[2], q2)), geo[3]);
      const float sy = rfa(rfa(rfa(rfm(geo[4], q0), rfm(geo[5], q1)), rfm(geo[6], q2)), geo[7]);
      const float dz = rfa(rfa(rfa(rfm(geo[8], q0), rfm(geo[9], q1)), rfm(geo[10], q2)), geo[11]);
      pts[i] = make_float4(rfa(half, __fdiv_rn(sx, dz)), rfa(half, __fdiv_rn(sy, dz)), dz, 0.f);
    }
  }
  __syncthreads();

  const int tile = blockIdx.x, ty = tile / tiles_x;
  const int px = (tile - ty * tiles_x) * RENDER_TILE + threadIdx.x, py = ty * RENDER_TILE + threadIdx.y;
  if (px >= p.S || py >= p.S) return;
  const float X = (float)px + 0.5f, Y = (float)py + 0.5f;
  float c[3];

  if (panel == 0) {
    // background: the video frame fitted into the panel (bilinear, edge-clamped), black without a video, white
    // outside the fitted rectangle
    const float u = rfs(__fdiv_rn(rfs(X, geo[13]), geo[12]), 0.5f);
    const float v = rfs(__fdiv_rn(rfs(Y, geo[14]), geo[12]), 0.5f);
    const bool inside = u >= -0.5f && u < rfs((float)p.Win, 0.5f) && v >= -0.5f && v < rfs((float)p.Hin, 0.5f);
    if (!inside) {
      c[0] = c[1] = c[2] = 255.f;
    } else if (!video) {
      c[0] = c[1] = c[2] = 0.f;
    } else {
      const float x0 = floorf(u), y0 = floorf(v);
      const float fx = rfs(u, x0), fy = rfs(v, y0), gx = rfs(1.f, fx), gy = rfs(1.f, fy);
      const int xa = min(max((int)x0, 0), p.Win - 1), xb = min(max((int)x0 + 1, 0), p.Win - 1);
      const int ya = min(max((int)y0, 0), p.Hin - 1), yb = min(max((int)y0 + 1, 0), p.Hin - 1);
      const unsigned char* im = video + g * p.video_frame;
      const unsigned char* r00 = im + ((long long)ya * p.Win + xa) * 3;
      const unsigned char* r01 = im + ((long long)ya * p.Win + xb) * 3;
      const unsigned char* r10 = im + ((long long)yb * p.Win + xa) * 3;
      const unsigned char* r11 = im + ((long long)yb * p.Win + xb) * 3;
      for (int ch = 0; ch < 3; ++ch) {
        const float top = rfa(rfm(gx, (float)r00[ch]), rfm(fx, (float)r01[ch]));
        const float bot = rfa(rfm(gx, (float)r10[ch]), rfm(fx, (float)r11[ch]));
        c[ch] = rfa(rfm(gy, top), rfm(fy, bot));
      }
    }
    // pink 2D bones: the largest coverage of any bone
    if (p.bones_2d) {
      float cov = 0.f;
      for (int m = 0; m < p.M; ++m)
        for (int j = 1; j < p.n_bones; ++j) {
          const int par = p.parents[j];
          if (par < 0) continue;
          const float4 a = pts[m * p.J + j], b = pts[m * p.J + par];
          float t;
          const float d = seg_dist(rfs(X, a.x), rfs(Y, a.y), rfs(b.x, a.x), rfs(b.y, a.y), &t);
          cov = fmaxf(cov, fminf(fmaxf(rfs(geo[16], d), 0.f), 1.f));
        }
      if (cov > 0.f) {
        c[0] = lerp_rn(c[0], 255.f, cov);
        c[1] = lerp_rn(c[1], 192.f, cov);
        c[2] = lerp_rn(c[2], 203.f, cov);
      }
    }
    // joint discs in scatter order (person-major), each a white ring around a black or red fill
    for (int i = 0; i < n_pts; ++i) {
      const float4 a = pts[i];
      const float dx = rfs(X, a.x), dy = rfs(Y, a.y);
      const float d = __fsqrt_rn(rfa(rfm(dx, dx), rfm(dy, dy)));
      const float co = fminf(fmaxf(rfs(geo[18], d), 0.f), 1.f);
      if (!(co > 0.f)) continue;
      const float ci = fminf(fmaxf(rfs(geo[17], d), 0.f), 1.f);
      const int j = i - (i / p.J) * p.J;
      const float red = ((p.right_mask >> j) & 1u) ? 255.f : 0.f;
      c[0] = lerp_rn(lerp_rn(c[0], 255.f, co), red, ci);
      c[1] = lerp_rn(lerp_rn(c[1], 255.f, co), 0.f, ci);
      c[2] = lerp_rn(lerp_rn(c[2], 255.f, co), 0.f, ci);
    }
  } else {
    // 3D panel: white, and the nearest covering bone (smallest interpolated depth; the first in order on a tie)
    c[0] = c[1] = c[2] = 255.f;
    float best_z = INFINITY, best_cov = 0.f;
    int best_j = -1;
    for (int e = 0; e < e_count; ++e)
      for (int j = 1; j < p.n_bones; ++j) {
        const int par = p.parents[j];
        if (par < 0) continue;
        const float4 a = pts[e * p.J + j], b = pts[e * p.J + par];
        float t;
        const float d = seg_dist(rfs(X, a.x), rfs(Y, a.y), rfs(b.x, a.x), rfs(b.y, a.y), &t);
        const float cov = rfs(geo[15], d);
        if (!(cov > 0.f)) continue;
        const float z = rfa(a.z, rfm(t, rfs(b.z, a.z)));
        if (z < best_z) {
          best_z = z;
          best_cov = fminf(cov, 1.f);
          best_j = j;
        }
      }
    if (best_j >= 0)
      for (int ch = 0; ch < 3; ++ch) c[ch] = lerp_rn(255.f, (float)p.color[best_j][ch], best_cov);
  }

  const int W = p.S * (1 + p.n_panel);
  unsigned char* o = out + ((f * p.S + py) * W + (long long)panel * p.S + px) * 3;
  for (int ch = 0; ch < 3; ++ch) o[ch] = (unsigned char)min(max(__float2int_rn(c[ch]), 0), 255);
}

// downsample_tensor (vis_h36m.py:53-55): out[o] = mean of in[o*factor .. o*factor+factor-1], element by element.
// float32 as numpy: a sequential float32 sum, then one float32 division; uint8 as numpy's mean of an integer array
// followed by astype('uint8'): the exact sum divided in double, truncated.
__global__ void downsample_f32_kernel(const float* __restrict__ x, long long n_out, long long row, int factor,
                                      float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_out * row) return;
  const long long o = idx / row, e = idx - o * row;
  const float* s = x + o * factor * row + e;
  float acc = s[0];
  for (int k = 1; k < factor; ++k) acc = __fadd_rn(acc, s[k * row]);
  out[idx] = __fdiv_rn(acc, (float)factor);
}

__global__ void downsample_u8_kernel(const unsigned char* __restrict__ x, long long n_out, long long row, int factor,
                                     unsigned char* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_out * row) return;
  const long long o = idx / row, e = idx - o * row;
  const unsigned char* s = x + o * factor * row + e;
  unsigned acc = 0;
  for (int k = 0; k < factor; ++k) acc += s[k * row];
  out[idx] = (unsigned char)((double)acc / (double)factor);
}

}  // namespace gast

// Host geometry of a call, in double and rounded once to float32 (DESIGN.md §8.5).
static void render_geometry(int S, double dpi, int Hin, int Win, double elev, double azim, double radius, double dist,
                            int shared, float* geo) {
  const double pi = 3.14159265358979323846;
  const double a = azim * pi / 180.0, e = elev * pi / 180.0;
  const double r[3] = {-sin(a), cos(a), 0.0};
  const double u[3] = {-sin(e) * cos(a), -sin(e) * sin(a), cos(e)};
  const double w[3] = {cos(e) * cos(a), cos(e) * sin(a), sin(e)};
  const double xy = shared ? radius : radius / 2;
  const double lo[3] = {-xy, -xy, 0.0}, hi[3] = {xy, xy, radius};
  const double h = sqrt(3.0) / 2;                             // the unit cube's half diagonal
  const double k = (S / 2.0) * (dist - h) / (h * dist);       // its bounding sphere just fits the panel
  double bx = 0, by = 0, bz = 1;
  for (int i = 0; i < 3; ++i) {
    const double span = hi[i] - lo[i], c = (lo[i] + hi[i]) / 2;
    const double ax = k * r[i] / span, ay = -k * u[i] / span, az = -w[i] / (dist * span);
    geo[i] = (float)ax;
    geo[4 + i] = (float)ay;
    geo[8 + i] = (float)az;
    bx -= ax * c;
    by -= ay * c;
    bz -= az * c;
  }
  geo[3] = (float)bx;
  geo[7] = (float)by;
  geo[11] = (float)bz;
  const bool wide = Win >= Hin;                               // the image fills the panel's width, else its height
  geo[12] = (float)(wide ? (double)S / Win : (double)S / Hin);
  geo[13] = (float)(wide ? 0.0 : S * (double)(Hin - Win) / (2.0 * Hin));
  geo[14] = (float)(wide ? S * (double)(Win - Hin) / (2.0 * Win) : 0.0);
  const double px = dpi / 72.0;                               // pixels per point
  const double rd = sqrt(10.0) / 2 * px, ew = 1.5 * px;       // scatter(s=10) disc radius, its 1.5 pt edge
  geo[15] = (float)(3.0 * px / 2 + 0.5);                      // 3D bones: linewidth 3
  geo[16] = (float)(1.5 * px / 2 + 0.5);                      // 2D bones: the default linewidth 1.5
  geo[17] = (float)(rd - ew / 2 + 0.5);
  geo[18] = (float)(rd + ew / 2 + 0.5);
  geo[19] = (float)(S / 2.0);
}

extern "C" int gast_render_geometry(int32_t S, float dpi, int32_t Hin, int32_t Win, float elev, float azim,
                                    float radius, float dist, int32_t shared, float* geo) {
  if (!geo || S < 8 || S > 8192 || !(dpi > 0.f) || Hin <= 0 || Win <= 0 || !(radius > 0.f) || !(dist > 1.f))
    return fail("gast_render_geometry: bad arguments (8 <= S <= 8192, dpi > 0, Hin, Win > 0, radius > 0, dist > 1)");
  render_geometry(S, dpi, Hin, Win, elev, azim, radius, dist, shared, geo);
  return 0;
}

extern "C" int gast_render_frames(const float* keypoints, int64_t n_kp_frames, int32_t M, int32_t J, const float* poses,
                                  int32_t n_pose, int64_t n_pose_frames, const uint8_t* video, int64_t n_video_frames,
                                  int32_t Hin, int32_t Win, const int32_t* parents, const uint8_t* colors,
                                  const int32_t* right, int32_t n_right, int32_t n_bones, int32_t S, float dpi,
                                  float elev, float azim, float radius, float dist, int32_t flags, int64_t f0,
                                  int32_t F, uint8_t* out, void* stream) {
  const int shared = flags & GAST_RENDER_SHARED_PANEL, follow = flags & GAST_RENDER_FOLLOW_ROOT;
  if (!keypoints || !poses || !parents || !colors || (n_right > 0 && !right) || !out || M <= 0 || J <= 0 ||
      J > RENDER_MAX_J || n_pose <= 0 || n_right < 0 || n_bones < 1 || n_bones > J || F <= 0 || f0 < 0 ||
      (flags & ~(GAST_RENDER_SHARED_PANEL | GAST_RENDER_FOLLOW_ROOT | GAST_RENDER_BONES_2D)))
    return fail("gast_render_frames: bad arguments");
  if ((long long)M * J > RENDER_MAX_PTS || (shared && (long long)n_pose * J > RENDER_MAX_PTS))
    return fail("gast_render_frames: %d x %d keypoints or %d shared poses exceed %d points", M, J, n_pose,
                RENDER_MAX_PTS);
  if (!shared && n_pose > RENDER_MAX_PANELS)
    return fail("gast_render_frames: %d 3D panels (at most %d)", n_pose, RENDER_MAX_PANELS);
  if (shared && follow) return fail("gast_render_frames: a shared panel cannot follow one pose's root");
  if (f0 + F > n_kp_frames || f0 + F > n_pose_frames || (video && f0 + F > n_video_frames))
    return fail("gast_render_frames: frames [%lld, %lld) exceed the inputs (%lld keypoint, %lld pose, %lld video frames)",
                (long long)f0, (long long)(f0 + F), (long long)n_kp_frames, (long long)n_pose_frames,
                (long long)(video ? n_video_frames : -1));
  RenderParams p;
  p.M = M;
  p.J = J;
  p.n_pose = n_pose;
  p.n_panel = shared ? 1 : n_pose;
  p.shared = shared ? 1 : 0;
  p.follow_root = follow ? 1 : 0;
  p.bones_2d = (flags & GAST_RENDER_BONES_2D) ? 1 : 0;
  p.n_bones = n_bones;
  p.S = S;
  p.Hin = Hin;
  p.Win = Win;
  p.kp_frame = (long long)M * J * 2;
  p.pose_stride = n_pose_frames * J * 3;
  p.video_frame = (long long)Hin * Win * 3;
  p.right_mask = 0;
  for (int j = 0; j < RENDER_MAX_J; ++j) {
    p.parents[j] = j < J ? parents[j] : -1;
    for (int ch = 0; ch < 3; ++ch) p.color[j][ch] = j < J ? colors[3 * j + ch] : 0;
    if (j < J && (p.parents[j] < -1 || p.parents[j] >= J))
      return fail("gast_render_frames: parents[%d] = %d is not -1 or a joint", j, p.parents[j]);
  }
  for (int i = 0; i < n_right; ++i) {
    if (right[i] < 0 || right[i] >= J) return fail("gast_render_frames: right joint %d out of range", right[i]);
    p.right_mask |= 1u << right[i];
  }
  if (gast_render_geometry(S, dpi, Hin, Win, elev, azim, radius, dist, shared, p.geo)) return 1;
  const int tiles = (int)cdiv(S, RENDER_TILE) * (int)cdiv(S, RENDER_TILE);
  const long long frame_bytes = (long long)S * S * (1 + p.n_panel) * 3;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (long long f = 0; f < F; f += 65535) {                     // grid.z bound
    const unsigned nf = (unsigned)std::min<long long>(65535, F - f);
    render_kernel<<<dim3(tiles, 1 + p.n_panel, nf), dim3(RENDER_TILE, RENDER_TILE), 0, st>>>(
        keypoints, poses, video, p, f0 + f, out + f * frame_bytes);
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_downsample_frames(const void* x, int64_t n_in_frames, int64_t frame_elems, int32_t factor,
                                      int32_t dtype, void* out, void* stream) {
  if (!x || !out || n_in_frames <= 0 || frame_elems <= 0 || factor < 1 || (dtype != 0 && dtype != 1))
    return fail("gast_downsample_frames: bad arguments (factor >= 1, dtype 0 = float32 or 1 = uint8)");
  const long long n_out = n_in_frames / factor, n = n_out * frame_elems;
  if (n_out == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (dtype == 0)
    downsample_f32_kernel<<<cdiv(n, 256), 256, 0, st>>>(reinterpret_cast<const float*>(x), n_out, frame_elems, factor,
                                                        reinterpret_cast<float*>(out));
  else
    downsample_u8_kernel<<<cdiv(n, 256), 256, 0, st>>>(reinterpret_cast<const unsigned char*>(x), n_out, frame_elems,
                                                       factor, reinterpret_cast<unsigned char*>(out));
  CUDA_OK(cudaGetLastError());
  return 0;
}
