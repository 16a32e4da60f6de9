// O(1)-per-frame streaming of the lifting network (SURVEY.md §8f N4; the reference's real-time path is a
// causal SpatioTemporalModelOptimized1f re-run on the last `receptive_field` frames for every new frame,
// gen_skes.py:43-69, tools/inference.py:19-110).  Included by gast_api.cu (uses its helpers).
//
// In the causal network every temporal stage i (filter width w_i, dilation d_i = w_0 ... w_{i-1}) maps its input
// sequence G_{i-1} to   S_i[t] = G_{i-1}[t] + f(G_{i-1}[t - (w_i-1) d_i], ..., G_{i-1}[t - d_i], G_{i-1}[t])
// (gast_net.py:139-143,167-174: with causal_shift = pad the residual slice and the last tap are both the newest
// position), and the blocks are pointwise in time.  So a pushed frame needs ONE new position per layer, given the
// layer inputs of the past: per stage a ring of R_i = w_i d_i slots holding G_{i-1}, slot = frame index mod R_i.
//
// Non-causal models (causal_shift = 0, gast_net.py:167-174,242-247).  Index every layer by the push that completes
// its window instead of by the frame it is centred on.  Then the taps are the same w_i positions t - (w_i-1) d_i ... t
// and the only change is the residual: the centre tap t - (w_i/2) d_i instead of the newest one.  So the rings, the
// tap rotation and the weights are shared with the causal form.  The one exception is the residual slot,
// (hs + R_i - (w_i/2) d_i) mod R_i.  The lags add up: the output of push t is the pose of frame t - pad, where
// pad = (rf-1)/2 (the latency).  The generator (common/generators.py:210-221) pads a sequence with pad copies of its
// first frame on the left and pad copies of its last frame on the right.
//   * Left: fill-fresh (below) gives a stream an infinite history of copies of its first frame.  The window of
//     frame t >= 0 reaches back to frame t - pad >= -pad, and that is all the left padding it sees.  The first `pad`
//     outputs after a start belong to frames before 0 and are dropped by the caller.
//   * Right: a HELD stream (`hold` mask) re-appends its own newest input frame instead of reading x.  After the last
//     frame, `pad` held pushes are exactly the right padding and return the last `pad` poses.  This also holds for
//     a sequence shorter than pad: a window then sees only padding beyond the sequence, as in the generator.
//
// Layout: rings are SLOT-major, ring_i[slot][stream][joint][channel], so that
//   * a slot is an ordinary contiguous (n_streams*J, C) activation matrix: the producing block writes it directly;
//   * the taps of stage i sit d_i slots apart: slots p, p + d_i, ..., p + (w_i-1) d_i with p = slot mod d_i -- a
//     fixed-stride gather, i.e. exactly the tap addressing the GEMM kernels already have (tap_stride), TMA-able.
// The taps appear in slot order, which is a ROTATION of time order (by r = slot div d_i): instead of moving data the
// stage's folded weights exist in w_i tap-rotated copies and the push picks copy r.  No activation is ever shifted.
//
// A stream's first frame replaces its whole history by copies of that frame (the edge padding of
// UnchunkedGenerator(pad, causal_shift = pad), common/generators.py:210-221).  With a constant history every layer
// input is constant in time, so it is enough to copy the freshly computed slot of each ring to the ring's other
// slots for those streams (stream_fill_fresh_kernel) before the stage reads its taps.
#pragma once

namespace gast {

// xhist (n, k0, J, F): the last k0 input frames of every stream, oldest first.  One thread per (stream, joint, feature).
// A held stream (hold[b] != 0, fresh[b] == 0) appends its own newest frame again and ignores x.
__global__ void stream_xpush_kernel(float* __restrict__ xhist, const float* __restrict__ x,
                                    const int32_t* __restrict__ fresh, const int32_t* __restrict__ hold, int n, int k0,
                                    int JF) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * JF) return;
  const int b = idx / JF, e = idx - b * JF;
  float* hrow = xhist + (long long)b * k0 * JF + e;
  const bool is_fresh = fresh && fresh[b];
  const float v = (hold && hold[b] && !is_fresh) ? hrow[(long long)(k0 - 1) * JF] : x[idx];
  if (is_fresh) {
    for (int k = 0; k < k0; ++k) hrow[(long long)k * JF] = v;
  } else {
    for (int k = 0; k + 1 < k0; ++k) hrow[(long long)k * JF] = hrow[(long long)(k + 1) * JF];
    hrow[(long long)(k0 - 1) * JF] = v;
  }
}

// ring (R, n, rowlen): for every fresh stream copy its row block of slot `src` to every other slot.
// grid = (n, chunks of the row block); a block whose stream is not fresh exits at once.
__global__ void stream_fill_fresh_kernel(float* __restrict__ ring, int R, int src, int n, long long rowlen,
                                         const int32_t* __restrict__ fresh) {
  const int b = blockIdx.x;
  if (!fresh[b]) return;
  const long long slot_stride = (long long)n * rowlen;
  const float4* s = reinterpret_cast<const float4*>(ring + (long long)src * slot_stride + (long long)b * rowlen);
  const long long n4 = rowlen >> 2;
  for (long long i = (long long)blockIdx.y * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.y * blockDim.x) {
    const float4 v = s[i];
    for (int r = 0; r < R; ++r)
      if (r != src) reinterpret_cast<float4*>(ring + (long long)r * slot_stride + (long long)b * rowlen)[i] = v;
  }
}

// ---- chunks of K frames per stream (gast_stream_push_chunk, below) ----
constexpr int CHUNK_XIN_THREADS = 256;

// xin (n, k0-1+K, J, F) = the last k0-1 frames of xhist followed by the K new frames x (n, K, J, F); then xhist = the
// last k0 frames of xin.  One block per stream.  hold (n, K) or null: a held frame (not fresh frame 0) repeats the
// stream's newest frame, which may be an earlier held frame of the chunk, so frame k takes x[b, src[k]] with src[k] the
// latest frame <= k that is not held (a block-wide max scan), or the newest frame of xhist when there is none.  A fresh
// stream's history is copies of its frame 0.  x rows of held frames are never read.  sidx (m) or null: row b of x / xin
// / fresh / hold belongs to state stream sidx[b] (a subset push, gast_stream_push_subset); null = stream b.  act (m) or
// null (all active): a row with act[b] == 0 sits the call out: its xin is built as if every frame were held (x is not
// read) and its input history is not written.
__global__ void __launch_bounds__(CHUNK_XIN_THREADS)
stream_chunk_xin_kernel(float* __restrict__ xhist, const float* __restrict__ x, float* __restrict__ xin,
                        const int32_t* __restrict__ fresh, const int32_t* __restrict__ hold, int k0, int K, int JF,
                        const int32_t* __restrict__ sidx, const int32_t* __restrict__ act) {
  __shared__ int src[CHUNK_XIN_THREADS];
  __shared__ int wmax[CHUNK_XIN_THREADS / 32];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool on = !act || act[b];
  const bool is_fresh = on && fresh && fresh[b];
  float* hrow = xhist + (long long)(sidx ? sidx[b] : b) * k0 * JF;
  float* irow = xin + (long long)b * (k0 - 1 + K) * JF;
  const float* xrow = x + (long long)b * K * JF;
  const int32_t* hb = hold ? hold + (long long)b * K : nullptr;
  int carry = -1;                                          // latest frame not held before this tile
  for (int t0 = 0; t0 < K; t0 += CHUNK_XIN_THREADS) {
    const int k = t0 + tid;
    const bool held = k >= K || !on || (hb && hb[k] && !(k == 0 && is_fresh));
    int v = held ? -1 : k;
    for (int o = 1; o < 32; o <<= 1) {                    // inclusive max scan: warp, then across warps
      const int u = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v = max(v, u);
    }
    if (lane == 31) wmax[warp] = v;
    __syncthreads();
    for (int w = 0; w < warp; ++w) v = max(v, wmax[w]);
    src[tid] = max(v, carry);
    __syncthreads();
    carry = src[CHUNK_XIN_THREADS - 1];
    const int nk = min(CHUNK_XIN_THREADS, K - t0);
    for (int e = tid; e < nk * JF; e += CHUNK_XIN_THREADS) {
      const int kk = e / JF, c = e - kk * JF, s = src[kk];
      irow[(long long)(k0 - 1 + t0 + kk) * JF + c] = s >= 0 ? xrow[(long long)s * JF + c] : hrow[(long long)(k0 - 1) * JF + c];
    }
    __syncthreads();                                       // src and wmax are rewritten by the next tile
  }
  for (int e = tid; e < (k0 - 1) * JF; e += CHUNK_XIN_THREADS)
    irow[e] = is_fresh ? xrow[e % JF] : hrow[e + JF];
  if (!on) return;                                         // the whole block: b is the block's row
  __syncthreads();                                         // every read of hrow is done; irow is visible to the block
  for (int e = tid; e < k0 * JF; e += CHUNK_XIN_THREADS) hrow[e] = irow[(long long)(K - 1) * JF + e];
}

// G (m, H+K, rowlen) = stage input at times step-H .. step+K-1: the head (positions p < H) from the ring slots
// (step - H + p) mod R, the tail (p >= H) from the previous block's K outputs tail (m, K, rowlen).  A fresh stream's head
// is copies of its tail position 0 (its history is constant, as stream_fill_fresh_kernel makes it).  The ring holds n
// streams per slot.  tab null: m = n, row b is stream b and hs = step mod R for all; else row b is state stream tab[b]
// at its own phase tab[m + b] (its step mod R_max, which R divides) and hs is unused.
__global__ void stream_chunk_gather_kernel(float4* __restrict__ G, const float4* __restrict__ ring,
                                           const float4* __restrict__ tail, const int32_t* __restrict__ fresh, int m,
                                           int n, int R, int hs, int H, int K, long long row4,
                                           const int32_t* __restrict__ tab) {
  const long long total = (long long)m * (H + K) * row4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long q = i % row4, f = i / row4;
    const int b = (int)(f / (H + K)), p = (int)(f - (long long)b * (H + K));
    float4 v;
    if (p >= H) v = tail[((long long)b * K + (p - H)) * row4 + q];
    else if (fresh && fresh[b]) v = tail[(long long)b * K * row4 + q];
    else {
      const int sb = tab ? tab[b] : b, h = tab ? tab[m + b] % R : hs;
      v = ring[((long long)((h - H + p + R) % R) * n + sb) * row4 + q];
    }
    G[i] = v;
  }
}

// Ring write-back after a chunk: slot p gets the stage input at the latest time t <= step+K-1 with t = p (mod R), from
// the tail of G when t falls in the chunk, copies of tail position 0 for a fresh stream, else the slot keeps its value.
// ek = (step + K - 1) mod R.  Launched after stream_chunk_gather_kernel, which reads slots this kernel overwrites.
// Grid over the R*m rows (slot, listed stream); tab as in stream_chunk_gather_kernel (null: m = n, ek for all; else
// ek = (tab[m + b] + K - 1) mod R per stream and slot p of stream tab[b] is written).  act (m) or null (all active):
// nothing is written for a row with act[b] == 0.
__global__ void stream_chunk_ring_kernel(float4* __restrict__ ring, const float4* __restrict__ G,
                                         const int32_t* __restrict__ fresh, int m, int n, int R, int ek, int H, int K,
                                         long long row4, const int32_t* __restrict__ tab,
                                         const int32_t* __restrict__ act) {
  const long long total = (long long)R * m * row4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long q = i % row4, f = i / row4;
    const int p = (int)(f / m), b = (int)(f - (long long)p * m);
    if (act && !act[b]) continue;
    const int e = tab ? (int)(((long long)tab[m + b] + K - 1) % R) : ek;
    const int k = K - 1 - (e - p + R) % R;                // chunk position of time t
    if (k < 0 && !(fresh && fresh[b])) continue;
    ring[tab ? ((long long)p * n + tab[b]) * row4 + q : i] = G[((long long)b * (H + K) + H + max(k, 0)) * row4 + q];
  }
}

// xin (n, k0-1+K, J, F) = the last k0-1 frames of xhist followed by K copies of its newest frame: the input of K held
// pushes (gast_stream_peek, below).  xhist is only read.  Grid-stride over the elements of xin.  sidx (m) or null: row b
// of xin is state stream sidx[b] (gast_stream_peek_subset); null = stream b.
__global__ void stream_peek_xin_kernel(const float* __restrict__ xhist, float* __restrict__ xin, int m, int k0, int K,
                                       int JF, const int32_t* __restrict__ sidx) {
  const int T = k0 - 1 + K;
  const long long total = (long long)m * T * JF;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long f = i / JF;
    const int e = (int)(i - f * JF), b = (int)(f / T), p = (int)(f - (long long)b * T);
    xin[i] = xhist[((long long)(sidx ? sidx[b] : b) * k0 + min(p + 1, k0 - 1)) * JF + e];
  }
}

// The table of a call driven by device-resident counts (gast_stream_push_device / _peek_device), over all n streams:
// tab[b] = b, tab[n + b] = phase = count mod rmax, tab[2n + b] = the effective fresh mask fresh[b] || count == 0 (a
// stream that never pushed starts a sequence: its ring is never read).  A negative count is taken as 0.  advance > 0 (a
// push) then sets the count of every active stream (act null: all) to count + advance.  Every value read here only
// selects a phase in [0, rmax) or a flag, so no content of counts, act or fresh can send a later kernel out of bounds.
__global__ void stream_device_table_kernel(int64_t* __restrict__ counts, const int32_t* __restrict__ act,
                                           const int32_t* __restrict__ fresh, int32_t* __restrict__ tab, int n,
                                           int64_t rmax, int advance) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < n; b += gridDim.x * blockDim.x) {
    const int64_t c = counts[b] > 0 ? counts[b] : 0;
    tab[b] = b;
    tab[n + b] = (int32_t)(c % rmax);
    tab[2 * n + b] = (fresh && fresh[b]) || c == 0;
    if (advance && (!act || act[b])) counts[b] = c + advance;
  }
}

// dst[n][k*Cw + c] = src[n][j*Cw + c],  j = (k - r - 1) mod taps: slot order -> time order of the taps
__global__ void rotate_taps_kernel(float* __restrict__ dst, const float* __restrict__ src, int N, int Cw, int taps, int r) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long K = (long long)taps * Cw;
  if (idx >= (long long)N * K) return;
  const long long nrow = idx / K;
  const int kc = (int)(idx - nrow * K);
  const int k = kc / Cw, c = kc - k * Cw;
  const int j = ((k - r - 1) % taps + taps) % taps;
  dst[idx] = src[nrow * K + (long long)j * Cw + c];
}

// ---- moving streams between states (gast_stream_export / gast_stream_import, below) ----
// A stream's snapshot is its history in time order: [xhist (k0, J, F)][ring_1 (R_1, J, C_1)] ... [ring_{L-1}], each
// part oldest first.  Part p is R_p rows of rowlen floats; row j of ring i of a stream at count c is its slot
// (c - R_i + j) mod R_i = (c + j) mod R_i, so the snapshot does not depend on the ring phase and an import at another
// count lands at that count's phase.  The input history is one row (it is kept in time order already).
struct MovePart { long long state_off, slot_stride, stream_stride, snap_off; int R, rowlen; };
struct MovePlan { MovePart part[GAST_MAX_STAGES]; int nparts; long long snap_floats; };

// grid = (rows of one snapshot, listed streams in a grid-stride loop); tab (2m): row b is state stream tab[b] at phase
// tab[m + b] (its count mod R_max, which every R_i divides).  kImport: snap (m, snap_floats) -> state, else the other
// way.  Plain float copies: the input history row (k0 J F floats) and the snapshot's part offsets need not be
// multiples of 4.
template <bool kImport>
__global__ void __launch_bounds__(256) stream_move_kernel(float* __restrict__ state, float* __restrict__ snap,
                                                          const MovePlan p, const int32_t* __restrict__ tab, int m) {
  int q = 0, j = blockIdx.x;
  while (j >= p.part[q].R) j -= p.part[q++].R;            // snapshot row -> (part, time position)
  const MovePart& g = p.part[q];
  for (int b = blockIdx.y; b < m; b += gridDim.y) {
    const int slot = q ? (tab[m + b] % g.R + j) % g.R : 0;
    float* s = state + g.state_off + slot * g.slot_stride + tab[b] * g.stream_stride;
    float* t = snap + b * p.snap_floats + g.snap_off + (long long)j * g.rowlen;
#pragma unroll 4
    for (int e = threadIdx.x; e < g.rowlen; e += blockDim.x) {
      if (kImport) s[e] = t[e];
      else t[e] = s[e];
    }
  }
}

}  // namespace gast

struct StreamPlan {
  int n = 0;
  std::vector<int> dil, R;              // per stage (index i-1): dilation d_i, ring slots R_i = w_i d_i
  std::vector<size_t> ring_off;         // float offsets into the state
  size_t xhist_off = 0, state_floats = 0;
};

static int stream_check(const gast_handle* h) {
  if (h->cfg.kind != GAST_KIND_MODEL) return fail("streaming is implemented for the MODEL kind only");
  if (h->cfg.dense) return fail("the dense ablation has no streaming form");
  // checked before a push touches the stream state (launch_expand checks it again for the forward)
  if (h->cfg.filter_widths[0] * h->cfg.in_features > EXP_MAXKF)
    return fail("expand: filter_width*in_features > %d unsupported", EXP_MAXKF);
  return 0;
}

static int stream_plan(const gast_handle* h, int n, StreamPlan* sp) {
  if (stream_check(h)) return 1;
  if (n <= 0) return fail("streaming: n_streams must be positive");
  const gast_cfg& c = h->cfg;
  const int J = c.num_joints, L = c.num_stages;
  sp->n = n;
  size_t off = 0;
  auto take = [&](size_t nf) { size_t o = off; off += (nf + 63) & ~(size_t)63; return o; };
  sp->xhist_off = take((size_t)n * c.filter_widths[0] * J * c.in_features);
  int d = c.filter_widths[0];
  for (int i = 1; i < L; ++i) {
    const int fw = c.filter_widths[i], Cw = c.channels << i;
    sp->dil.push_back(d);
    sp->R.push_back(fw * d);
    sp->ring_off.push_back(take((size_t)fw * d * n * J * Cw));
    d *= fw;
  }
  sp->state_floats = off;
  return 0;
}

extern "C" size_t gast_stream_state_bytes(gast_t* h, int32_t n_streams) {
  if (!h) return 0;
  StreamPlan sp;
  if (stream_plan(h, n_streams, &sp)) return 0;
  return sp.state_floats * sizeof(float) + 256;
}

struct StreamBufs { float *E, *tmp, *act, *fin; BlockBufs bb; };

static void stream_bufs(const gast_handle* h, int n, Arena& a, StreamBufs* sb) {
  const int J = h->cfg.num_joints, C = h->cfg.channels, L = h->cfg.num_stages;
  const size_t rows = (size_t)n * J;
  const int Cmax = C << (L - 1);                 // widest block input
  sb->E = a.take(rows * C);
  sb->tmp = a.take(rows * Cmax);
  sb->act = a.take(rows * Cmax);
  sb->fin = a.take(rows * 2 * Cmax);
  sb->bb.XY = a.take(rows * 2 * Cmax); sb->bb.L = a.take(rows * Cmax); sb->bb.AB = a.take(rows * 8);
  sb->bb.Y = a.take(rows * Cmax); sb->bb.Gl = a.take(rows * Cmax);
}

extern "C" size_t gast_stream_workspace_bytes(gast_t* h, int32_t n_streams) {
  if (!h || stream_check(h) || n_streams <= 0) return 0;
  Arena a{nullptr, 0, 0, true};
  StreamBufs sb;
  stream_bufs(h, n_streams, a, &sb);
  return a.off + 256;
}

// tap-rotated copies of the folded temporal-conv weights (+ their tensor-core hi/lo splits); rebuilt after every gast_prepare
static int stream_prepare(gast_handle* h, cudaStream_t st) {
  for (size_t i = 0; i < h->stages.size(); ++i) {
    StageConsts& s = h->stages[i];
    const int fw = h->cfg.filter_widths[i + 1];
    if (s.taps != fw) return fail("streaming: stage %zu has %d taps, expected %d", i, s.taps, fw);
    if ((int)s.Wrot.size() != fw) {
      s.Wrot.assign(fw, nullptr);
      s.tc_rot.assign(fw, TcWeights());
      for (int r = 0; r < fw; ++r)
        if (dalloc(h, &s.Wrot[r], (size_t)s.Cw * fw * s.Cw)) return 1;
    }
    const long long tot = (long long)s.Cw * fw * s.Cw;
    for (int r = 0; r < fw; ++r) {
      rotate_taps_kernel<<<cdiv(tot, 256), 256, 0, st>>>(s.Wrot[r], s.Wt, s.Cw, s.Cw, fw, r);
      if (prep_one_tc(h, st, s.tc_rot[r], s.Wrot[r], s.Cw, fw * s.Cw)) return 1;
    }
  }
  CUDA_OK(cudaGetLastError());
  h->stream_ready = true;
  return 0;
}

extern "C" int32_t gast_stream_latency(const gast_t* h) {
  if (!h || stream_check(h)) return -1;
  return h->cfg.causal ? 0 : (gast_receptive_field(h) - 1) / 2;
}

extern "C" int gast_stream_push_ex(gast_t* h, void* state, int64_t step, const float* x, float* y, int32_t n_streams,
                                   const int32_t* fresh, const int32_t* hold, void* workspace, size_t workspace_bytes,
                                   void* stream) {
  if (!h) return fail("gast_stream_push_ex: null handle");
  if (step < 0 || !state || !x || !y) return fail("gast_stream_push_ex: bad arguments");
  StreamPlan sp;
  if (stream_plan(h, n_streams, &sp)) return 1;
  if (!h->prepared) return fail("gast_stream_push_ex: gast_prepare() has not run since the last gast_bind()");
  if (call_begin(h, "gast_stream_push_ex", gast_stream_workspace_bytes(h, n_streams), workspace, workspace_bytes))
    return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!h->stream_ready && stream_prepare(h, st)) return 1;
  const gast_cfg& c = h->cfg;
  const int n = n_streams, J = c.num_joints, C = c.channels, L = c.num_stages, k0 = c.filter_widths[0], Fin = c.in_features;
  float* sbase = reinterpret_cast<float*>(align256(state));
  Arena a = workspace_arena(workspace, workspace_bytes);
  StreamBufs sb;
  stream_bufs(h, n, a, &sb);
  const long long rows = (long long)n * J;
  // input history + expand (gast_net.py:163-164) on the last k0 frames
  float* xhist = sbase + sp.xhist_off;
  stream_xpush_kernel<<<cdiv((long long)n * J * Fin, 256), 256, 0, st>>>(xhist, x, fresh, hold, n, k0, J * Fin);
  h->launches++;
  if (launch_expand(h, st, xhist, sb.E, rows, k0, 1, 1)) return 1;
  auto slot_ptr = [&](int i /*stage 1..L-1*/) {
    const int R = sp.R[i - 1], Cw = C << i;
    return sbase + sp.ring_off[i - 1] + (size_t)(step % R) * n * J * Cw;
  };
  float* bout = (L > 1) ? slot_ptr(1) : sb.fin;
  if (run_block(h, st, h->blocks[0], sb.E, n, sb.bb, bout)) return 1;
  for (int i = 1; i < L; ++i) {
    StageConsts& s = h->stages[i - 1];
    const int Cw = s.Cw, fw = c.filter_widths[i], d = sp.dil[i - 1], R = sp.R[i - 1];
    float* ring = sbase + sp.ring_off[i - 1];
    const int hs = (int)(step % R);
    const long long slot_floats = (long long)n * J * Cw;
    if (fresh) {
      dim3 g((unsigned)n, (unsigned)std::max<long long>(1, std::min<long long>(8, (long long)J * Cw / 4 / 256)));
      stream_fill_fresh_kernel<<<g, 256, 0, st>>>(ring, R, hs, n, (long long)J * Cw, fresh);
      h->launches++;
    }
    // taps = slots p0 + k d with the weights rotated to slot order; residual = the newest slot (causal_shift = pad)
    // or the centre tap (causal_shift = 0)
    const int p0 = hs % d, r = hs / d;
    const int rs = c.causal ? hs : (hs + R - (fw / 2) * d) % R;
    const RowMap same{n, n, 1, 0};
    const ASeg taps = seg_taps(ring + (long long)p0 * slot_floats, Cw, Cw, fw, (long long)d * slot_floats, same);
    if (run_stage(h, st, s, n, taps, s.Wrot[r], &s.tc_rot[r], sb.tmp, ring + (long long)rs * slot_floats, same, sb.act))
      return 1;
    bout = (i < L - 1) ? slot_ptr(i + 1) : sb.fin;
    if (run_block(h, st, h->blocks[i], sb.act, n, sb.bb, bout)) return 1;
  }
  if (launch_shrink(h, st, bout, y, rows, nullptr, nullptr)) return 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_stream_push(gast_t* h, void* state, int64_t step, const float* x, float* y, int32_t n_streams,
                                const int32_t* fresh, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h) return fail("gast_stream_push: null handle");
  if (h->cfg.kind == GAST_KIND_MODEL && !h->cfg.causal)
    return fail("gast_stream_push needs a causal model (gen_skes.py:59: causal=True): a non-causal network has no "
                "output for the newest frame (gast_stream_push_ex returns it `latency` pushes later)");
  return gast_stream_push_ex(h, state, step, x, y, n_streams, fresh, nullptr, workspace, workspace_bytes, stream);
}

// ---- K frames per stream in one call ---------------------------------------------------------------------------
// gast_stream_push_chunk is gast_stream_push_ex at steps step .. step+K-1 with x[:, k], fresh at k = 0 only and
// hold[:, k], run as ONE forward over n*K positions on the dilated schedule's kernels.  Temporal stage i (width w,
// dilation d, ring R = w d) needs its last H = (w-1) d inputs before the chunk plus the K new ones: they are gathered
// into G (n, H+K, J, Cw) (head from the ring, tail from the previous block), the stage runs on G with the time-ordered
// weights Wt and the row map of the whole-sequence forward (taps d*J*Cw floats apart, residual at the newest or the
// centre tap), and every ring slot is then given the input of the latest time it stands for, so that the next push
// (single or chunk) finds the history it expects.  The blocks are pointwise in time and run on n*K frames.
struct ChunkBufs { float *xin, *G; StreamBufs sb; int32_t* tab; };

// The workspace of a chunk call over m streams of K frames: the chunk buffers, then `table` ints per stream: 0 for a
// lockstep call, 2 for the (stream, phase) table of a subset call (gast_stream_push_subset below), 3 for the (stream,
// phase, fresh) table of a device-counts call (gast_stream_push_device).  sp gives the dilations only.
static int chunk_bufs(const gast_handle* h, const StreamPlan& sp, int m, int K, int table, const char* who, Arena& a,
                      ChunkBufs* cb) {
  const gast_cfg& c = h->cfg;
  const int J = c.num_joints, k0 = c.filter_widths[0];
  if (K < 1) return fail("%s: K must be at least 1 (got %d)", who, K);
  if ((long long)m * K * J >= 0x7fffffffLL) return fail("expand: more than 2^31 positions in one call");
  size_t g = 0;
  for (int i = 1; i < c.num_stages; ++i)
    g = std::max(g, (size_t)m * ((c.filter_widths[i] - 1) * sp.dil[i - 1] + K) * J * (c.channels << i));
  cb->xin = a.take((size_t)m * (k0 - 1 + K) * J * c.in_features);
  cb->G = a.take(g);
  stream_bufs(h, m * K, a, &cb->sb);
  cb->tab = table ? reinterpret_cast<int32_t*>(a.take((size_t)table * m)) : nullptr;
  return 0;
}

// Bytes that chunk_bufs takes (0 after a refusal): what the workspace of the call must hold.
static size_t chunk_workspace_bytes(const gast_handle* h, const StreamPlan& sp, int m, int K, int table,
                                    const char* who) {
  Arena dry{nullptr, 0, 0, true};
  ChunkBufs cb;
  return chunk_bufs(h, sp, m, K, table, who, dry, &cb) ? 0 : dry.off + 256;
}

extern "C" size_t gast_stream_chunk_workspace_bytes(gast_t* h, int32_t n_streams, int32_t K) {
  StreamPlan sp;
  if (!h || stream_plan(h, n_streams, &sp)) return 0;
  return chunk_workspace_bytes(h, sp, n_streams, K, 0, "gast_stream_chunk_workspace_bytes");
}

// The chunk forward after its input frames are in cb.xin: expand, block 0, the temporal stages on their gathered
// history (ring write-back when write_rings), shrink into y (m, K, J, 3).  tab null: all m = sp.n streams at `step`;
// else the device table of a subset call (stream_chunk_gather_kernel): m listed streams, each at its own phase.  act
// (m) or null: the write-back skips the rows with act[b] == 0.
static int chunk_forward(gast_handle* h, cudaStream_t st, const StreamPlan& sp, float* sbase, int64_t step, int m,
                         int K, const int32_t* fresh, bool write_rings, const ChunkBufs& cb, float* y,
                         const int32_t* tab, const int32_t* act) {
  const gast_cfg& c = h->cfg;
  const int n = sp.n, J = c.num_joints, L = c.num_stages, k0 = c.filter_widths[0];
  const long long F = (long long)m * K;                  // frames of the chunk, in (stream, frame) order
  const StreamBufs& sb = cb.sb;
  if (launch_expand(h, st, cb.xin, sb.E, F * J, k0 - 1 + K, K, 1)) return 1;
  if (run_block(h, st, h->blocks[0], sb.E, F, sb.bb, sb.fin)) return 1;
  const unsigned grid_cap = (unsigned)h->sm_count * 16;
  for (int i = 1; i < L; ++i) {
    const StageConsts& s = h->stages[i - 1];
    const int Cw = s.Cw, fw = c.filter_widths[i], d = sp.dil[i - 1], R = sp.R[i - 1], H = (fw - 1) * d;
    if (s.taps != fw) return fail("streaming: stage %d has %d taps, expected %d", i - 1, s.taps, fw);
    if ((J * Cw) % 4) return fail("streaming chunk: J*channels of stage %d is not a multiple of 4", i);
    float* ring = sbase + sp.ring_off[i - 1];
    const long long row4 = (long long)J * Cw / 4;
    const long long g4 = (long long)m * (H + K) * row4, r4 = (long long)R * m * row4;
    stream_chunk_gather_kernel<<<(unsigned)std::min<long long>(cdiv(g4, 256), grid_cap), 256, 0, st>>>(
        reinterpret_cast<float4*>(cb.G), reinterpret_cast<const float4*>(ring),
        reinterpret_cast<const float4*>(sb.fin), fresh, m, n, R, (int)(step % R), H, K, row4, tab);
    h->launches++;
    if (write_rings) {
      stream_chunk_ring_kernel<<<(unsigned)std::min<long long>(cdiv(r4, 256), grid_cap), 256, 0, st>>>(
          reinterpret_cast<float4*>(ring), reinterpret_cast<const float4*>(cb.G), fresh, m, n, R,
          (int)((step + K - 1) % R), H, K, row4, tab, act);
      h->launches++;
    }
    // output frame (b, t) = time step+t: taps at G positions t, t+d, ..., t+H; residual at the newest tap (causal)
    // or the centre tap t + H - (w/2) d (non-causal), as in the whole-sequence forward
    const ASeg taps = seg_taps(cb.G, Cw, Cw, fw, (long long)d * J * Cw, RowMap{K, H + K, 1, 0});
    const RowMap res{K, H + K, 1, c.causal ? H : H - (fw / 2) * d};
    if (run_stage(h, st, s, F, taps, s.Wt, &s.tc_t, sb.tmp, cb.G, res, sb.act)) return 1;
    if (run_block(h, st, h->blocks[i], sb.act, F, sb.bb, sb.fin)) return 1;
  }
  // rows of fin are already in (stream, frame, joint) order
  if (launch_shrink(h, st, sb.fin, y, F * J, nullptr, nullptr)) return 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- any subset of the streams, each at its own frame count -------------------------------------------------------
// A subset call runs the chunk (or peek) forward over the m listed streams only: the four copy kernels read and write
// the state rows of stream streams[i] at that stream's own ring phase, and everything between them (expand, blocks,
// stages on the time-ordered weights Wt, shrink) works on the m*K gathered frames as for a chunk.  Every ring size R_i
// divides the largest one, R_max = w_0 w_1 ... w_{L-1} (R_i = w_i d_i and d_{i+1} = R_i), so one phase per stream,
// steps[i] mod R_max, gives its slot in every ring.  The (stream, phase) table goes to the workspace in one copy.
extern "C" size_t gast_stream_subset_workspace_bytes(gast_t* h, int32_t m, int32_t K) {
  StreamPlan sp;                                           // the chunk buffers of m streams
  if (!h || m < 1 || stream_plan(h, m, &sp)) return 0;
  return chunk_workspace_bytes(h, sp, m, K, 2, "gast_stream_subset_workspace_bytes");
}

// Host-side checks of a subset call and its table: {streams[i]} then {steps[i] mod R_max}.  *lockstep = the call lists
// every stream in order at one step (the chunk path's own call, no table needed).
static int subset_table(const StreamPlan& sp, const int32_t* streams, const int64_t* steps,
                        int m, int64_t min_step, const char* who, std::vector<int32_t>* tab, bool* lockstep) {
  const int n = sp.n;
  if (m < 1 || m > n) return fail("%s: m must be in [1, n_streams = %d] (got %d)", who, n, m);
  const int64_t Rmax = sp.R.empty() ? 1 : sp.R.back();
  std::vector<char> seen(n, 0);
  tab->resize((size_t)2 * m);
  *lockstep = m == n;
  for (int i = 0; i < m; ++i) {
    const int32_t s = streams[i];
    if (s < 0 || s >= n) return fail("%s: streams[%d] = %d is outside [0, %d)", who, i, s, n);
    if (seen[s]) return fail("%s: stream %d is listed twice", who, s);
    seen[s] = 1;
    if (steps[i] < min_step) return fail("%s: steps[%d] = %lld must be at least %lld", who, i, (long long)steps[i],
                                         (long long)min_step);
    (*tab)[i] = s;
    (*tab)[m + i] = (int32_t)(steps[i] % Rmax);
    *lockstep = *lockstep && s == i && steps[i] == steps[0];
  }
  return 0;
}

// ---- the four chunk entries ---------------------------------------------------------------------------------------
// One chunk call over m streams of K frames.  x null: a peek (below), every frame held and the state only read, its
// input built by stream_peek_xin_kernel; else a push of x through stream_chunk_xin_kernel.  streams null: the lockstep
// form, all m = n_streams streams at `step`; else the subset form, stream streams[i] at steps[i], which takes the
// lockstep addressing (no table) when it lists every stream in order at one step.  counts (device) instead of streams:
// the device-counts form, all m = n_streams streams at their own counts, the ones with active[b] == 0 (active null:
// none) sitting the call out; its table is built on the device by stream_device_table_kernel.  Every refusal comes
// before the first launch.
static int chunk_call(const char* who, gast_handle* h, void* state, int n_streams, const int32_t* streams,
                      const int64_t* steps, int64_t* counts, const int32_t* active, int64_t step, int m, int K,
                      const float* x, float* y, const int32_t* fresh, const int32_t* hold, void* workspace,
                      size_t workspace_bytes, void* stream) {
  if (!h) return fail("%s: null handle", who);
  const bool peek = !x;
  const int table = streams ? 2 : counts ? 3 : 0;                // ints per stream in the workspace table
  if (peek) {
    const int32_t lat = gast_stream_latency(h);
    if (lat < 0) return 1;
    if (lat == 0)
      return fail("%s needs a non-causal model: a causal model returns the pose of the pushed frame, so none is ever "
                  "pending", who);
    if (K < 1 || K > lat) return fail("%s: K must be in [1, latency = %d] (got %d)", who, lat, K);
    if (!table && step < 1) return fail("%s: step must be at least 1 (the state holds no pushed frame)", who);
  }
  if ((!table && step < 0) || !state || !y) return fail("%s: bad arguments", who);
  StreamPlan sp;
  if (stream_plan(h, n_streams, &sp)) return 1;
  std::vector<int32_t> tab;
  bool lockstep = !counts;
  if (streams && subset_table(sp, streams, steps, m, peek ? 1 : 0, who, &tab, &lockstep)) return 1;
  const size_t need = chunk_workspace_bytes(h, sp, m, K, table, who);
  if (need == 0) return 1;
  if (!h->prepared) return fail("%s: gast_prepare() has not run since the last gast_bind()", who);
  if (call_begin(h, who, need, workspace, workspace_bytes)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int J = h->cfg.num_joints, k0 = h->cfg.filter_widths[0], JF = J * h->cfg.in_features;
  float* sbase = reinterpret_cast<float*>(align256(state));
  Arena a = workspace_arena(workspace, workspace_bytes);
  ChunkBufs cb;
  chunk_bufs(h, sp, m, K, table, who, a, &cb);                   // sized above: cannot fail
  const int32_t* dtab = nullptr;
  if (counts) {                                                  // the table and the effective fresh mask
    stream_device_table_kernel<<<(unsigned)std::min<long long>(cdiv(m, 256), h->sm_count), 256, 0, st>>>(
        counts, active, fresh, cb.tab, m, sp.R.empty() ? 1 : sp.R.back(), peek ? 0 : K);
    h->launches++;
    dtab = cb.tab;
    fresh = cb.tab + 2 * m;
  } else if (!lockstep) {
    CUDA_OK(cudaMemcpyAsync(cb.tab, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
    dtab = cb.tab;
  }
  if (streams) step = steps[0];                                  // read by the lockstep addressing only
  if (peek) {
    const long long xe = (long long)m * (k0 - 1 + K) * JF;
    stream_peek_xin_kernel<<<(unsigned)std::min<long long>(cdiv(xe, 256), (long long)h->sm_count * 16), 256, 0, st>>>(
        sbase + sp.xhist_off, cb.xin, m, k0, K, JF, dtab);
  } else {
    stream_chunk_xin_kernel<<<m, CHUNK_XIN_THREADS, 0, st>>>(sbase + sp.xhist_off, x, cb.xin, fresh, hold, k0, K, JF,
                                                             dtab, active);
  }
  h->launches++;
  return chunk_forward(h, st, sp, sbase, step, m, K, fresh, !peek, cb, y, dtab, active);
}

extern "C" int gast_stream_push_chunk(gast_t* h, void* state, int64_t step, const float* x, float* y, int32_t n_streams,
                                      int32_t K, const int32_t* fresh, const int32_t* hold, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  if (!x) return fail("gast_stream_push_chunk: bad arguments");   // a null x would make the call a peek
  return chunk_call("gast_stream_push_chunk", h, state, n_streams, nullptr, nullptr, nullptr, nullptr, step, n_streams,
                    K, x, y, fresh, hold, workspace, workspace_bytes, stream);
}

// ---- peek: the poses K held pushes would return, without pushing ------------------------------------------------
// gast_stream_peek is gast_stream_push_chunk with fresh = null and every frame held, minus every write to the state:
// stream_peek_xin_kernel builds the chunk input from the input history without updating it, and the stages gather
// their ring history but write no slot back.  Row k of stream s is the pose the (k+1)-th held push would return: for a
// sequence of l pushed frames, the pose of frame l - latency + k with the generator's right padding applied after
// frame l - 1.
extern "C" int gast_stream_peek(gast_t* h, const void* state, int64_t step, float* y, int32_t n_streams, int32_t K,
                                void* workspace, size_t workspace_bytes, void* stream) {
  // only read: chunk_forward writes no ring back for a peek
  return chunk_call("gast_stream_peek", h, const_cast<void*>(state), n_streams, nullptr, nullptr, nullptr, nullptr, step,
                    n_streams, K, nullptr, y, nullptr, nullptr, workspace, workspace_bytes, stream);
}

extern "C" int gast_stream_push_subset(gast_t* h, void* state, int32_t n_streams, const int32_t* streams,
                                       const int64_t* steps, int32_t m, int32_t K, const float* x, float* y,
                                       const int32_t* fresh, const int32_t* hold, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  const char* who = "gast_stream_push_subset";
  if (!streams || !steps) return fail("%s: null streams or steps", who);   // null streams is the lockstep form
  if (!x) return fail("%s: bad arguments", who);
  return chunk_call(who, h, state, n_streams, streams, steps, nullptr, nullptr, 0, m, K, x, y, fresh, hold, workspace,
                    workspace_bytes, stream);
}

extern "C" int gast_stream_peek_subset(gast_t* h, const void* state, int32_t n_streams, const int32_t* streams,
                                       const int64_t* steps, int32_t m, int32_t K, float* y, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  const char* who = "gast_stream_peek_subset";
  if (!streams || !steps) return fail("%s: null streams or steps", who);
  return chunk_call(who, h, const_cast<void*>(state), n_streams, streams, steps, nullptr, nullptr, 0, m, K, nullptr, y,
                    nullptr, nullptr, workspace, workspace_bytes, stream);
}

// ---- the frame counts on the device: calls a CUDA graph can capture ----------------------------------------------
// The subset entries read the streams and their counts on the host and copy the table from host memory, so a captured
// call would replay the phases of the tick it was captured at.  These keep the counts on the device: one small kernel
// (stream_device_table_kernel) turns counts and the active mask into the subset table of all n streams, then the chunk
// path runs as for a subset call listing every stream, with the inactive rows built as held rows and left out of every
// state write.  No argument depends on the step, and every check is on the host, before the first launch.
extern "C" size_t gast_stream_device_workspace_bytes(gast_t* h, int32_t n_streams, int32_t K) {
  StreamPlan sp;
  if (!h || stream_plan(h, n_streams, &sp)) return 0;
  return chunk_workspace_bytes(h, sp, n_streams, K, 3, "gast_stream_device_workspace_bytes");
}

extern "C" int gast_stream_push_device(gast_t* h, void* state, int32_t n_streams, int64_t* counts,
                                       const int32_t* active, int32_t K, const float* x, float* y,
                                       const int32_t* fresh, const int32_t* hold, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  const char* who = "gast_stream_push_device";
  if (!counts) return fail("%s: null counts", who);
  if (!x) return fail("%s: bad arguments", who);                 // a null x would make the call a peek
  return chunk_call(who, h, state, n_streams, nullptr, nullptr, counts, active, 0, n_streams, K, x, y, fresh, hold,
                    workspace, workspace_bytes, stream);
}

extern "C" int gast_stream_peek_device(gast_t* h, const void* state, int32_t n_streams, const int64_t* counts,
                                       const int32_t* active, int32_t K, float* y, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  const char* who = "gast_stream_peek_device";
  if (!counts) return fail("%s: null counts", who);
  // only read: the table kernel advances no count for a peek, and chunk_forward writes no ring back
  return chunk_call(who, h, const_cast<void*>(state), n_streams, nullptr, nullptr, const_cast<int64_t*>(counts), active,
                    0, n_streams, K, nullptr, y, nullptr, nullptr, workspace, workspace_bytes, stream);
}

// ---- moving streams between states: a gather to and a scatter from their time-ordered snapshots -----------------
// The parts of a snapshot (stream_move_kernel) over the state layout of stream_plan.
static MovePlan move_plan(const gast_handle* h, const StreamPlan& sp) {
  const gast_cfg& c = h->cfg;
  const int J = c.num_joints, xrow = c.filter_widths[0] * J * c.in_features;
  MovePlan p{};
  p.part[0] = MovePart{(long long)sp.xhist_off, 0, xrow, 0, 1, xrow};
  long long off = xrow;
  for (size_t i = 0; i < sp.R.size(); ++i) {
    const int row = J * (c.channels << (i + 1)), R = sp.R[i];
    p.part[i + 1] = MovePart{(long long)sp.ring_off[i], (long long)sp.n * row, row, off, R, row};
    off += (long long)R * row;
  }
  p.nparts = (int)sp.R.size() + 1;
  p.snap_floats = off;
  return p;
}

extern "C" size_t gast_stream_snapshot_floats(gast_t* h) {
  StreamPlan sp;
  if (!h || stream_plan(h, 1, &sp)) return 0;
  return (size_t)move_plan(h, sp).snap_floats;
}

extern "C" size_t gast_stream_move_workspace_bytes(gast_t* h, int32_t m) {
  if (!h || stream_check(h) || m < 1) return 0;
  Arena a{nullptr, 0, 0, true};
  a.take((size_t)2 * m);                                   // the (stream, phase) table, 2 int32 per stream
  return a.off + 256;
}

// Both directions: the subset entries' checks of streams and counts (counts >= 1), the table to the workspace in one
// copy, then one stream_move_kernel launch.  Every refusal comes before the first launch.
static int move_call(const char* who, bool import, gast_handle* h, void* state, int n_streams, const int32_t* streams,
                     const int64_t* counts, int m, float* snap, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h) return fail("%s: null handle", who);
  if (!streams || !counts) return fail("%s: null streams or counts", who);
  if (!state || !snap) return fail("%s: bad arguments", who);
  StreamPlan sp;
  if (stream_plan(h, n_streams, &sp)) return 1;
  std::vector<int32_t> tab;
  bool lockstep;
  if (subset_table(sp, streams, counts, m, 1, who, &tab, &lockstep)) return 1;
  if (call_begin(h, who, gast_stream_move_workspace_bytes(h, m), workspace, workspace_bytes)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const MovePlan p = move_plan(h, sp);
  int32_t* dtab = reinterpret_cast<int32_t*>(workspace_arena(workspace, workspace_bytes).take((size_t)2 * m));
  CUDA_OK(cudaMemcpyAsync(dtab, tab.data(), tab.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  int rows = 0;
  for (int q = 0; q < p.nparts; ++q) rows += p.part[q].R;
  const dim3 grid((unsigned)rows, (unsigned)std::min(m, 65535));
  float* sbase = reinterpret_cast<float*>(align256(state));
  if (import) stream_move_kernel<true><<<grid, 256, 0, st>>>(sbase, snap, p, dtab, m);
  else stream_move_kernel<false><<<grid, 256, 0, st>>>(sbase, snap, p, dtab, m);
  h->launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_stream_export(gast_t* h, const void* state, int32_t n_streams, const int32_t* streams,
                                  const int64_t* counts, int32_t m, float* out, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  // only read: the export kernel writes the snapshot
  return move_call("gast_stream_export", false, h, const_cast<void*>(state), n_streams, streams, counts, m, out,
                   workspace, workspace_bytes, stream);
}

extern "C" int gast_stream_import(gast_t* h, void* state, int32_t n_streams, const int32_t* streams,
                                  const int64_t* counts, int32_t m, const float* in, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  // only read: the import kernel reads the snapshot
  return move_call("gast_stream_import", true, h, state, n_streams, streams, counts, m, const_cast<float*>(in),
                   workspace, workspace_bytes, stream);
}
