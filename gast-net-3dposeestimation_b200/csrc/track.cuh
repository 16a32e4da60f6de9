// SORT (lib/track/sort.py) on the device: the Kalman box trackers, the IoU association, scipy's
// linear_sum_assignment and the tracker list's births and deaths, for a chunk of frames of many videos in one launch.
//
// One CTA runs one sequence (one video, or one camera), its frames one after the other.  The sequence's state (frame
// count, next id, the ordered tracker list, each tracker's fp64 x[7] and P[7x7] and its counters) lives in the
// caller's buffer; the CTA copies it into shared memory at the start of the launch and back at the end.  Inside a
// frame the work is parallel over trackers (one warp per tracker for the predict and the update, the 7x7 products
// spread over its lanes) and over the IoU entries; the assignment is scipy's shortest-augmenting-path solver
// (rectangular_lsap.cpp) run by one warp, its Dijkstra scan split over the lanes and reduced with scipy's own choice
// rule; the list bookkeeping is one thread's.  Nothing is ordered by atomics, so calls repeat bit for bit.
//
// Arithmetic (DESIGN.md §8.8): the measurement z and the detection's area are float32 as the reference computes them,
// everything else fp64; the IoU, z, the predict and every H product are explicit round-to-nearest intrinsics in the
// reference's order, so they are bit-exact; S^-1 and the products with K are fp64 in a fixed order.
//
// Included at the end of gast_api.cu (uses fail / CUDA_OK).
#pragma once
#include <math.h>

namespace gast {

constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int SORT_SCRATCH = 128;            // doubles of update scratch per warp: y, S, S^-1, K, (I - KH) P
constexpr int SORT_MAX_SMEM = 227 * 1024;    // opt-in shared memory per block on sm_90
constexpr int SORT_MAX_CAPACITY = 4096;
constexpr long long SORT_MAGIC = 0x54524f53;  // "SORT"
// status bits (include/gast_b200.h)
constexpr int SORT_ST_COUNT = 1, SORT_ST_CAPACITY = 2, SORT_ST_IOU = 4, SORT_ST_INF = 8, SORT_ST_STATE = 16;
// header words of a sequence's state
enum { SH_FRAME = 0, SH_NEXT_ID, SH_NTRK, SH_STATUS, SH_MAX_AGE, SH_MIN_HITS, SH_CAPACITY, SH_MAGIC, SH_WORDS };

__host__ __device__ inline size_t sort_align(size_t b) { return (b + 15) & ~(size_t)15; }

// one sequence's state: the header, then the list and per-tracker arrays indexed by slot
struct SortLayout {
  size_t order, freestk, tsu, hits, streak, age, id, x, P, bytes;
  __host__ __device__ explicit SortLayout(int cap) {
    size_t o = SH_WORDS * sizeof(long long);
    order = o;   o = sort_align(o + (size_t)cap * 4);
    freestk = o; o = sort_align(o + (size_t)cap * 4);
    tsu = o;     o = sort_align(o + (size_t)cap * 4);
    hits = o;    o = sort_align(o + (size_t)cap * 4);
    streak = o;  o = sort_align(o + (size_t)cap * 4);
    age = o;     o = sort_align(o + (size_t)cap * 4);
    id = o;      o = sort_align(o + (size_t)cap * 8);
    x = o;       o = sort_align(o + (size_t)cap * 8 * sizeof(double));
    P = o;       o = sort_align(o + (size_t)cap * 49 * sizeof(double));
    bytes = o;
  }
};

// the launch's scratch after the state image: frame detections, predicted boxes, association and solver arrays
struct SortScratch {
  size_t dets, pbox, flag, upd, dmatch, births, outpos, u, v, spc, path, col4row, row4col, remaining, SR, SC, warp,
      bytes;
  __host__ __device__ SortScratch(size_t base, int cap, int max_det) {
    const int L = cap > max_det ? cap : max_det;
    size_t o = base;
    dets = o;      o = sort_align(o + (size_t)max_det * 16);
    pbox = o;      o = sort_align(o + (size_t)cap * 32);
    flag = o;      o = sort_align(o + (size_t)cap * 4);
    upd = o;       o = sort_align(o + (size_t)cap * 4);
    dmatch = o;    o = sort_align(o + (size_t)max_det * 4);
    births = o;    o = sort_align(o + (size_t)max_det * 4);
    outpos = o;    o = sort_align(o + (size_t)cap * 4);
    u = o;         o = sort_align(o + (size_t)L * 8);
    v = o;         o = sort_align(o + (size_t)L * 8);
    spc = o;       o = sort_align(o + (size_t)L * 8);
    path = o;      o = sort_align(o + (size_t)L * 4);
    col4row = o;   o = sort_align(o + (size_t)L * 4);
    row4col = o;   o = sort_align(o + (size_t)L * 4);
    remaining = o; o = sort_align(o + (size_t)L * 4);
    SR = o;        o = sort_align(o + (size_t)L);
    SC = o;        o = sort_align(o + (size_t)L);
    warp = o;      o = sort_align(o + (size_t)SORT_WARPS * SORT_SCRATCH * 8);
    bytes = o;
  }
};

inline size_t sort_smem_bytes(int cap, int max_det) {
  const SortLayout lo(cap);
  return SortScratch(lo.bytes, cap, max_det).bytes;
}

// np.maximum / np.minimum on scalars: NaN in either operand gives NaN
__device__ __forceinline__ double sort_max(double a, double b) { return (a >= b || a != a) ? a : b; }
__device__ __forceinline__ double sort_min(double a, double b) { return (a <= b || a != a) ? a : b; }

// sort.py's numba iou(det, trk) stored into the float32 matrix: the detection's area in float32, the rest in fp64.
// *ok is false where the reference raises: a zero denominator (numba's ZeroDivisionError) or an entry
// linear_sum_assignment refuses (NaN, or -inf after the negation; +inf is refused with it).
__device__ __forceinline__ float sort_iou(const float4 d, const double4 t, bool* ok) {
  const double xx1 = sort_max((double)d.x, t.x), yy1 = sort_max((double)d.y, t.y);
  const double xx2 = sort_min((double)d.z, t.z), yy2 = sort_min((double)d.w, t.w);
  const double w = sort_max(0.0, __dsub_rn(xx2, xx1)), h = sort_max(0.0, __dsub_rn(yy2, yy1));
  const double wh = __dmul_rn(w, h);
  const float ad = __fmul_rn(__fsub_rn(d.z, d.x), __fsub_rn(d.w, d.y));
  const double at = __dmul_rn(__dsub_rn(t.z, t.x), __dsub_rn(t.w, t.y));
  const double den = __dsub_rn(__dadd_rn((double)ad, at), wh);
  const float o = __double2float_rn(__ddiv_rn(wh, den));
  *ok = den != 0.0 && isfinite(o);
  return o;
}

// convert_x_to_bbox in fp64
__device__ __forceinline__ double4 sort_x_to_box(const double* x) {
  const double w = __dsqrt_rn(__dmul_rn(x[2], x[3]));
  const double h = __ddiv_rn(x[2], w);
  const double w2 = __ddiv_rn(w, 2.0), h2 = __ddiv_rn(h, 2.0);
  return make_double4(__dsub_rn(x[0], w2), __dsub_rn(x[1], h2), __dadd_rn(x[0], w2), __dadd_rn(x[1], h2));
}

// convert_bbox_to_z of a float32 box: float32 throughout (w / float(h) stays float32 under NumPy 2)
__device__ __forceinline__ float4 sort_z(const float4 b) {
  const float w = __fsub_rn(b.z, b.x), h = __fsub_rn(b.w, b.y);
  return make_float4(__fadd_rn(b.x, __fdiv_rn(w, 2.f)), __fadd_rn(b.y, __fdiv_rn(h, 2.f)), __fmul_rn(w, h),
                     __fdiv_rn(w, h));
}

__device__ __forceinline__ double sort_Q(int i, int j) {
  if (i != j) return 0.0;
  return i < 4 ? 1.0 : (i < 6 ? 0.01 : __dmul_rn(0.01, 0.01));
}
__device__ __forceinline__ double sort_R(int k) { return k < 2 ? 1.0 : 10.0; }

// KalmanBoxTracker.predict's filter step for one tracker, by one warp: the x[6] guard, x = Fx, P = F P F' + Q.  F is
// 0/1, so each entry is one or two two-term sums, rounded as any BLAS order rounds them.
__device__ __forceinline__ void sort_predict(double* x, double* P, int lane) {
  const double x2 = x[2];
  double x6 = x[6];
  if (__dadd_rn(x6, x2) <= 0.0) x6 = __dmul_rn(x6, 0.0);
  double xn = 0.0;
  if (lane < 7) {
    const double xi = lane == 6 ? x6 : x[lane];
    xn = lane < 3 ? __dadd_rn(xi, lane == 2 ? x6 : x[lane + 4]) : xi;
  }
  double pn[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int e = lane + 32 * r;
    pn[r] = 0.0;
    if (e < 49) {
      const int i = e / 7, j = e % 7;
      double a = P[e];
      if (i < 3) a = __dadd_rn(a, P[e + 28]);
      if (j < 3) {
        double b = P[e + 4];
        if (i < 3) b = __dadd_rn(b, P[e + 32]);
        a = __dadd_rn(a, b);
      }
      pn[r] = __dadd_rn(a, sort_Q(i, j));
    }
  }
  __syncwarp();
  if (lane < 7) x[lane] = xn;
  if (lane < 49 - 32) P[lane + 32] = pn[1];
  P[lane] = pn[0];
  __syncwarp();
}

// KalmanFilter.update (filterpy 1.4.5) for one tracker by one warp: y = z - Hx, S = HPH' + R, K = PH'S^-1, x += Ky,
// P = (I - KH) P (I - KH)' + K R K'.  H selects x[0..3], so y, PH' and S are exact; S^-1 (Gauss-Jordan, S is
// symmetric positive definite) and the products with K are fp64 in a fixed order.  sc: the warp's scratch.
__device__ __forceinline__ void sort_update(double* x, double* P, const float4 z, double* sc, int lane) {
  double* y = sc;          // 4
  double* S = sc + 4;      // 16, reduced in place
  double* SI = sc + 20;    // 16
  double* K = sc + 36;     // 28
  double* M = sc + 64;     // 49
  if (lane < 4) y[lane] = __dsub_rn((double)(lane == 0 ? z.x : lane == 1 ? z.y : lane == 2 ? z.z : z.w), x[lane]);
  if (lane < 16) {
    const int a = lane >> 2, b = lane & 3;
    S[lane] = __dadd_rn(P[a * 7 + b], a == b ? sort_R(a) : 0.0);
    SI[lane] = a == b ? 1.0 : 0.0;
  }
  __syncwarp();
  if (lane == 0) {
    for (int c = 0; c < 4; ++c) {
      const double inv = 1.0 / S[c * 4 + c];
      for (int k = 0; k < 4; ++k) {
        S[c * 4 + k] *= inv;
        SI[c * 4 + k] *= inv;
      }
      for (int r = 0; r < 4; ++r) {
        if (r == c) continue;
        const double f = S[r * 4 + c];
        for (int k = 0; k < 4; ++k) {
          S[r * 4 + k] -= f * S[c * 4 + k];
          SI[r * 4 + k] -= f * SI[c * 4 + k];
        }
      }
    }
  }
  __syncwarp();
  if (lane < 28) {
    const int i = lane >> 2, j = lane & 3;
    double k = 0.0;
    for (int t = 0; t < 4; ++t) k += P[i * 7 + t] * SI[t * 4 + j];
    K[lane] = k;
  }
  __syncwarp();
  double xn = 0.0;
  if (lane < 7) {
    xn = x[lane];
    double ky = 0.0;
    for (int j = 0; j < 4; ++j) ky += K[lane * 4 + j] * y[j];
    xn += ky;
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int e = lane + 32 * r;
    if (e < 49) {
      const int i = e / 7, j = e % 7;
      double m = 0.0;
      for (int t = 0; t < 7; ++t) {
        const double ikh = (i == t ? 1.0 : 0.0) - (t < 4 ? K[i * 4 + t] : 0.0);
        m += ikh * P[t * 7 + j];
      }
      M[e] = m;
    }
  }
  __syncwarp();
  if (lane < 7) x[lane] = xn;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int e = lane + 32 * r;
    if (e < 49) {
      const int i = e / 7, j = e % 7;
      double p = 0.0;
      for (int t = 0; t < 7; ++t) {
        const double ikh = (j == t ? 1.0 : 0.0) - (t < 4 ? K[j * 4 + t] : 0.0);
        p += M[i * 7 + t] * ikh;
      }
      double q = 0.0;
      for (int t = 0; t < 4; ++t) q += K[i * 4 + t] * sort_R(t) * K[j * 4 + t];
      P[e] = p + q;
    }
  }
  __syncwarp();
}

struct SortShared {
  long long* hdr;
  int *order, *freestk, *tsu, *hits, *streak, *age;
  long long* id;
  double *x, *P;
  float4* dets;
  double4* pbox;
  int *flag, *upd, *dmatch, *births, *outpos;
  double *u, *v, *spc;
  int *path, *col4row, *row4col, *remaining;
  unsigned char *SR, *SC;
  double* warp;
};

// -(float32 iou) as linear_sum_assignment's fp64 cost of row i, column j of the (possibly transposed) matrix
__device__ __forceinline__ double sort_cost(const SortShared& s, bool tr, int i, int j) {
  bool ok;
  const float o = tr ? sort_iou(s.dets[j], s.pbox[i], &ok) : sort_iou(s.dets[i], s.pbox[j], &ok);
  return (double)(-o);
}

// scipy 1.18's linear_sum_assignment(cost) (rectangular_lsap.cpp) on the n x m cost matrix -iou, by one warp.
// Rows are the detections, columns the trackers; a tall matrix is solved transposed, as scipy does.  The Dijkstra
// scan is split over the lanes; the reduction keeps scipy's choice: the lowest reduced cost, among equal costs the
// last unassigned column in `remaining` order if there is one, else the first.  Leaves dmatch[d] = the tracker
// position matched to detection d, or -1.
__device__ __forceinline__ void sort_lsap(const SortShared& s, int n, int m, int lane) {
  const bool tr = m < n;
  const int nr = tr ? m : n, nc = tr ? n : m;
  for (int j = lane; j < nc; j += 32) {
    s.v[j] = 0.0;
    s.row4col[j] = -1;
    s.path[j] = -1;
  }
  for (int i = lane; i < nr; i += 32) {
    s.u[i] = 0.0;
    s.col4row[i] = -1;
  }
  __syncwarp();
  for (int cur = 0; cur < nr; ++cur) {
    for (int j = lane; j < nc; j += 32) {
      s.remaining[j] = nc - j - 1;
      s.SC[j] = 0;
      s.spc[j] = INFINITY;
    }
    for (int i = lane; i < nr; i += 32) s.SR[i] = 0;
    __syncwarp();
    double minVal = 0.0;
    int num_remaining = nc, i = cur, sink = -1;
    while (sink == -1) {
      if (lane == 0) s.SR[i] = 1;
      double lowest = INFINITY;
      int key = -1;       // unassigned: nc + it (the last wins), assigned: nc - 1 - it (the first wins)
      const double ui = s.u[i];
      for (int it = lane; it < num_remaining; it += 32) {
        const int j = s.remaining[it];
        const double r = __dsub_rn(__dsub_rn(__dadd_rn(minVal, sort_cost(s, tr, i, j)), ui), s.v[j]);
        double c = s.spc[j];
        if (r < c) {
          s.path[j] = i;
          s.spc[j] = c = r;
        }
        const int k = s.row4col[j] == -1 ? nc + it : nc - 1 - it;
        if (c < lowest || (c == lowest && k > key)) {
          lowest = c;
          key = k;
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double ol = __shfl_xor_sync(0xffffffffu, lowest, o);
        const int ok = __shfl_xor_sync(0xffffffffu, key, o);
        if (ol < lowest || (ol == lowest && ok > key)) {
          lowest = ol;
          key = ok;
        }
      }
      minVal = lowest;
      const int index = key >= nc ? key - nc : nc - 1 - key;
      __syncwarp();
      const int j = s.remaining[index];
      if (s.row4col[j] == -1)
        sink = j;
      else
        i = s.row4col[j];
      __syncwarp();
      if (lane == 0) {
        s.SC[j] = 1;
        s.remaining[index] = s.remaining[num_remaining - 1];
      }
      --num_remaining;
      __syncwarp();
    }
    if (lane == 0) s.u[cur] = __dadd_rn(s.u[cur], minVal);
    for (int r = lane; r < nr; r += 32)
      if (s.SR[r] && r != cur) s.u[r] = __dadd_rn(s.u[r], __dsub_rn(minVal, s.spc[s.col4row[r]]));
    for (int c = lane; c < nc; c += 32)
      if (s.SC[c]) s.v[c] = __dsub_rn(s.v[c], __dsub_rn(minVal, s.spc[c]));
    __syncwarp();
    if (lane == 0) {
      int j = sink;
      while (true) {
        const int r = s.path[j];
        s.row4col[j] = r;
        const int t = s.col4row[r];
        s.col4row[r] = j;
        j = t;
        if (r == cur) break;
      }
    }
    __syncwarp();
  }
  for (int d = lane; d < n; d += 32) s.dmatch[d] = -1;
  __syncwarp();
  if (tr) {
    for (int t = lane; t < nr; t += 32) s.dmatch[s.col4row[t]] = t;
  } else {
    for (int d = lane; d < nr; d += 32) s.dmatch[d] = s.col4row[d];
  }
}

__device__ __forceinline__ void sort_birth(const SortShared& s, int slot, const float4 b, long long id) {
  const float4 z = sort_z(b);
  double* x = s.x + (size_t)slot * 8;
  double* P = s.P + (size_t)slot * 49;
  x[0] = z.x;
  x[1] = z.y;
  x[2] = z.z;
  x[3] = z.w;
  x[4] = x[5] = x[6] = 0.0;
  for (int e = 0; e < 49; ++e) P[e] = (e % 8 == 0) ? (e < 32 ? 10.0 : 10000.0) : 0.0;
  s.tsu[slot] = 0;
  s.hits[slot] = 0;
  s.streak[slot] = 0;
  s.age[slot] = 0;
  s.id[slot] = id;
}

__global__ void sort_init_kernel(unsigned char* state, int cap, int max_age, int min_hits,
                                 const long long* __restrict__ first_ids) {
  const SortLayout lo(cap);
  unsigned char* st = state + (size_t)blockIdx.x * lo.bytes;
  long long* hdr = reinterpret_cast<long long*>(st);
  int* freestk = reinterpret_cast<int*>(st + lo.freestk);
  int* order = reinterpret_cast<int*>(st + lo.order);
  for (int k = threadIdx.x; k < cap; k += blockDim.x) {
    freestk[k] = cap - 1 - k;    // popped from the top: slot 0 first
    order[k] = -1;
  }
  if (threadIdx.x == 0) {
    hdr[SH_FRAME] = 0;
    hdr[SH_NEXT_ID] = first_ids ? first_ids[blockIdx.x] : 0;
    hdr[SH_NTRK] = 0;
    hdr[SH_STATUS] = 0;
    hdr[SH_MAX_AGE] = max_age;
    hdr[SH_MIN_HITS] = min_hits;
    hdr[SH_CAPACITY] = cap;
    hdr[SH_MAGIC] = SORT_MAGIC;
  }
}

__global__ void __launch_bounds__(SORT_THREADS)
sort_update_kernel(unsigned char* __restrict__ state, int cap, int K, const float* __restrict__ boxes,
                   const int* __restrict__ counts, int max_det, int skip_empty, double* __restrict__ out_rows,
                   int* __restrict__ out_counts, int* __restrict__ status_out) {
  extern __shared__ __align__(16) unsigned char sort_smem[];
  __shared__ int sh_nb, sh_any;
  const SortLayout lo(cap);
  const SortScratch sl(lo.bytes, cap, max_det);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint4* gst = reinterpret_cast<uint4*>(state + (size_t)blockIdx.x * lo.bytes);
  uint4* sst = reinterpret_cast<uint4*>(sort_smem);
  for (size_t k = tid; k < lo.bytes / 16; k += SORT_THREADS) sst[k] = gst[k];
  SortShared s;
  s.hdr = reinterpret_cast<long long*>(sort_smem);
  s.order = reinterpret_cast<int*>(sort_smem + lo.order);
  s.freestk = reinterpret_cast<int*>(sort_smem + lo.freestk);
  s.tsu = reinterpret_cast<int*>(sort_smem + lo.tsu);
  s.hits = reinterpret_cast<int*>(sort_smem + lo.hits);
  s.streak = reinterpret_cast<int*>(sort_smem + lo.streak);
  s.age = reinterpret_cast<int*>(sort_smem + lo.age);
  s.id = reinterpret_cast<long long*>(sort_smem + lo.id);
  s.x = reinterpret_cast<double*>(sort_smem + lo.x);
  s.P = reinterpret_cast<double*>(sort_smem + lo.P);
  s.dets = reinterpret_cast<float4*>(sort_smem + sl.dets);
  s.pbox = reinterpret_cast<double4*>(sort_smem + sl.pbox);
  s.flag = reinterpret_cast<int*>(sort_smem + sl.flag);
  s.upd = reinterpret_cast<int*>(sort_smem + sl.upd);
  s.dmatch = reinterpret_cast<int*>(sort_smem + sl.dmatch);
  s.births = reinterpret_cast<int*>(sort_smem + sl.births);
  s.outpos = reinterpret_cast<int*>(sort_smem + sl.outpos);
  s.u = reinterpret_cast<double*>(sort_smem + sl.u);
  s.v = reinterpret_cast<double*>(sort_smem + sl.v);
  s.spc = reinterpret_cast<double*>(sort_smem + sl.spc);
  s.path = reinterpret_cast<int*>(sort_smem + sl.path);
  s.col4row = reinterpret_cast<int*>(sort_smem + sl.col4row);
  s.row4col = reinterpret_cast<int*>(sort_smem + sl.row4col);
  s.remaining = reinterpret_cast<int*>(sort_smem + sl.remaining);
  s.SR = sort_smem + sl.SR;
  s.SC = sort_smem + sl.SC;
  s.warp = reinterpret_cast<double*>(sort_smem + sl.warp);
  __syncthreads();
  if (tid == 0 && s.hdr[SH_STATUS] == 0 && (s.hdr[SH_MAGIC] != SORT_MAGIC || s.hdr[SH_CAPACITY] != cap))
    s.hdr[SH_STATUS] = SORT_ST_STATE;
  __syncthreads();
  const int max_age = (int)s.hdr[SH_MAX_AGE], min_hits = (int)s.hdr[SH_MIN_HITS];

  for (int t = 0; t < K; ++t) {
    const long long fr = (long long)blockIdx.x * K + t;
    const int n_in = counts[fr];
    const int n = (n_in < 0 || n_in > max_det) ? 0 : n_in;
    int nz = 0;
    const float* fb = boxes + fr * max_det * 4;
    for (int k = tid; k < 4 * n; k += SORT_THREADS) {
      const float b = fb[k];
      reinterpret_cast<float*>(s.dets)[k] = b;
      nz |= b != 0.f;                                       // NaN counts as nonzero, as ndarray.any() does
    }
    const int any = __syncthreads_or(nz);
    if (s.hdr[SH_STATUS] != 0 || n != n_in) {
      __syncthreads();
      if (tid == 0) {
        if (s.hdr[SH_STATUS] == 0) s.hdr[SH_STATUS] = SORT_ST_COUNT;
        out_counts[fr] = 0;
      }
      __syncthreads();
      continue;
    }
    if (skip_empty && (n == 0 || !any)) {
      if (tid == 0) out_counts[fr] = -1;
      continue;                                             // no update call: frame_count stays
    }

    // 1. predict every tracker (warp per tracker), then drop the NaN ones in list order
    int ntrk = (int)s.hdr[SH_NTRK];
    for (int k = warp; k < ntrk; k += SORT_WARPS) {
      const int slot = s.order[k];
      double* x = s.x + (size_t)slot * 8;
      sort_predict(x, s.P + (size_t)slot * 49, lane);
      if (lane == 0) {
        s.age[slot] += 1;
        if (s.tsu[slot] > 0) s.streak[slot] = 0;
        s.tsu[slot] += 1;
        const double4 b = sort_x_to_box(x);
        s.pbox[k] = b;
        const bool nan = isnan(b.x) || isnan(b.y) || isnan(b.z) || isnan(b.w);
        const bool inf = isinf(b.x) || isinf(b.y) || isinf(b.z) || isinf(b.w);
        s.flag[k] = nan ? 1 : (inf ? 2 : 0);
      }
    }
    __syncthreads();
    if (tid == 0) {
      s.hdr[SH_FRAME] += 1;
      int w = 0, nfree = cap - ntrk;
      for (int k = 0; k < ntrk; ++k) {
        if (s.flag[k] == 2) s.hdr[SH_STATUS] = SORT_ST_INF;   // masked out of trks, kept in self.trackers
        if (s.flag[k] == 1) {
          s.freestk[nfree++] = s.order[k];
        } else {
          s.order[w] = s.order[k];
          s.pbox[w] = s.pbox[k];
          ++w;
        }
      }
      s.hdr[SH_NTRK] = w;
    }
    __syncthreads();
    ntrk = (int)s.hdr[SH_NTRK];

    // 2. the IoU matrix must be one linear_sum_assignment accepts
    if (s.hdr[SH_STATUS] == 0 && ntrk > 0 && n > 0) {
      int bad = 0;
      for (int e = tid; e < n * ntrk; e += SORT_THREADS) {
        bool ok;
        sort_iou(s.dets[e / ntrk], s.pbox[e % ntrk], &ok);
        bad |= !ok;
      }
      if (__syncthreads_or(bad) && tid == 0) s.hdr[SH_STATUS] = SORT_ST_IOU;
      __syncthreads();
    }
    if (s.hdr[SH_STATUS] != 0) {
      __syncthreads();
      if (tid == 0) out_counts[fr] = 0;
      __syncthreads();
      continue;
    }

    // 3. the assignment, then births and updates as associate_detections_to_trackers orders them
    for (int k = tid; k < ntrk; k += SORT_THREADS) s.upd[k] = -1;
    if (ntrk > 0 && n > 0) {
      if (warp == 0) sort_lsap(s, n, ntrk, lane);
    } else {
      for (int d = tid; d < n; d += SORT_THREADS) s.dmatch[d] = -1;
    }
    __syncthreads();
    if (tid == 0) {
      int nb = 0;
      for (int d = 0; d < n; ++d)
        if (s.dmatch[d] < 0) s.births[nb++] = d;              // unmatched detections, in detection order
      for (int d = 0; d < n; ++d) {                           // then the low-IoU matches, in matched row order
        const int k = s.dmatch[d];
        if (k < 0) continue;
        bool ok;
        if (sort_iou(s.dets[d], s.pbox[k], &ok) < 0.3f)
          s.births[nb++] = d;
        else
          s.upd[k] = d;
      }
      sh_nb = nb;
    }
    __syncthreads();
    for (int k = warp; k < ntrk; k += SORT_WARPS) {
      const int d = s.upd[k];
      if (d < 0) continue;
      const int slot = s.order[k];
      sort_update(s.x + (size_t)slot * 8, s.P + (size_t)slot * 49, sort_z(s.dets[d]), s.warp + warp * SORT_SCRATCH,
                  lane);
      if (lane == 0) {
        s.tsu[slot] = 0;
        s.hits[slot] += 1;
        s.streak[slot] += 1;
      }
    }
    __syncthreads();
    if (tid == 0) {
      const int nb = sh_nb;
      if (ntrk + nb > cap) {
        s.hdr[SH_STATUS] = SORT_ST_CAPACITY;
      } else {
        for (int b = 0; b < nb; ++b) {
          const int slot = s.freestk[cap - ntrk - 1];
          s.order[ntrk++] = slot;
          sort_birth(s, slot, s.dets[s.births[b]], s.hdr[SH_NEXT_ID]++);
        }
        s.hdr[SH_NTRK] = ntrk;
      }
      // 4. the output rows: the list reversed, filtered
      int c = 0;
      const long long fc = s.hdr[SH_FRAME];
      for (int k = ntrk - 1; k >= 0; --k) {
        const int slot = s.order[k];
        s.outpos[k] = (s.tsu[slot] < 1 && (s.streak[slot] >= min_hits || fc <= min_hits)) ? c++ : -1;
      }
      sh_any = c;
    }
    __syncthreads();
    if (s.hdr[SH_STATUS] != 0) {
      if (tid == 0) out_counts[fr] = 0;
      __syncthreads();
      continue;
    }
    ntrk = (int)s.hdr[SH_NTRK];
    for (int k = tid; k < ntrk; k += SORT_THREADS) {
      const int p = s.outpos[k];
      if (p < 0) continue;
      const int slot = s.order[k];
      const double4 b = sort_x_to_box(s.x + (size_t)slot * 8);
      double* o = out_rows + ((size_t)fr * cap + p) * 5;
      o[0] = b.x;
      o[1] = b.y;
      o[2] = b.z;
      o[3] = b.w;
      o[4] = (double)(s.id[slot] + 1);
    }
    __syncthreads();
    // 5. the dead trackers leave, the rest keep their order
    if (tid == 0) {
      out_counts[fr] = sh_any;
      int w = 0, nfree = cap - ntrk;
      for (int k = 0; k < ntrk; ++k) {
        const int slot = s.order[k];
        if (s.tsu[slot] > max_age)
          s.freestk[nfree++] = slot;
        else
          s.order[w++] = slot;
      }
      s.hdr[SH_NTRK] = w;
    }
    __syncthreads();
  }

  __syncthreads();
  for (size_t k = tid; k < lo.bytes / 16; k += SORT_THREADS) gst[k] = sst[k];
  if (tid == 0) status_out[blockIdx.x] = (int)s.hdr[SH_STATUS];
}

}  // namespace gast

extern "C" size_t gast_sort_state_bytes(int32_t S, int32_t capacity) {
  using namespace gast;
  if (S < 0 || capacity < 1 || capacity > SORT_MAX_CAPACITY) {
    fail("gast_sort_state_bytes: S = %d, capacity = %d (1 .. %d)", S, capacity, SORT_MAX_CAPACITY);
    return 0;
  }
  return (size_t)(S > 0 ? S : 1) * SortLayout(capacity).bytes;
}

extern "C" int gast_sort_init(void* state, int32_t S, int32_t capacity, int32_t max_age, int32_t min_hits,
                              const int64_t* first_ids, void* stream) {
  using namespace gast;
  if (!state || S < 0 || capacity < 1 || capacity > SORT_MAX_CAPACITY || max_age < 0 || min_hits < 0)
    return fail("gast_sort_init: bad arguments (S = %d, capacity = %d (1 .. %d), max_age = %d, min_hits = %d)", S,
                capacity, SORT_MAX_CAPACITY, max_age, min_hits);
  if (S == 0) return 0;
  sort_init_kernel<<<S, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<unsigned char*>(state), capacity, max_age, min_hits,
      reinterpret_cast<const long long*>(first_ids));
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_sort_update(void* state, int32_t S, int32_t capacity, int32_t K, const float* boxes,
                                const int32_t* counts, int32_t max_det, int32_t flags, double* out_rows,
                                int32_t* out_counts, int32_t* status, void* stream) {
  using namespace gast;
  if (!state || !counts || !out_counts || !status || S < 0 || K < 0 || max_det < 0 || flags < 0 || flags > 1 ||
      capacity < 1 || capacity > SORT_MAX_CAPACITY || (!boxes && max_det > 0) || !out_rows)
    return fail("gast_sort_update: bad arguments (flags: GAST_SORT_SKIP_EMPTY; capacity 1 .. %d)", SORT_MAX_CAPACITY);
  const size_t smem = sort_smem_bytes(capacity, max_det);
  if (smem > (size_t)SORT_MAX_SMEM)
    return fail("gast_sort_update: capacity %d with max_det %d needs %zu bytes of shared memory (at most %d)", capacity,
                max_det, smem, SORT_MAX_SMEM);
  if (S == 0) return 0;
  CUDA_OK(cudaFuncSetAttribute(sort_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sort_update_kernel<<<S, SORT_THREADS, smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<unsigned char*>(state), capacity, K, boxes, counts, max_det, flags & 1, out_rows, out_counts,
      status);
  CUDA_OK(cudaGetLastError());
  return 0;
}
