// O(1)-per-frame causal streaming of the lifting network (SURVEY.md §8f N4; the reference's real-time path is a
// causal SpatioTemporalModelOptimized1f re-run on the last `receptive_field` frames for every new frame,
// gen_skes.py:43-69, tools/inference.py:19-110).  Included by gast_api.cu (uses its helpers).
//
// In the causal network every temporal stage i (filter width w_i, dilation d_i = w_0 ... w_{i-1}) maps its input
// sequence G_{i-1} to   S_i[t] = G_{i-1}[t] + f(G_{i-1}[t - (w_i-1) d_i], ..., G_{i-1}[t - d_i], G_{i-1}[t])
// (gast_net.py:139-143,167-174: with causal_shift = pad the residual slice and the last tap are both the newest
// position), and the blocks are pointwise in time.  So a pushed frame needs ONE new position per layer, given the
// layer inputs of the past: per stage a ring of R_i = w_i d_i slots holding G_{i-1}, slot = frame index mod R_i.
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
__global__ void stream_xpush_kernel(float* __restrict__ xhist, const float* __restrict__ x,
                                    const int32_t* __restrict__ fresh, int n, int k0, int JF) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * JF) return;
  const int b = idx / JF, e = idx - b * JF;
  float* hrow = xhist + (long long)b * k0 * JF + e;
  const float v = x[idx];
  if (fresh && fresh[b]) {
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

}  // namespace gast

struct StreamPlan {
  int n = 0;
  std::vector<int> dil, R;              // per stage (index i-1): dilation d_i, ring slots R_i = w_i d_i
  std::vector<size_t> ring_off;         // float offsets into the state
  size_t xhist_off = 0, state_floats = 0;
};

static int stream_check(const gast_handle* h) {
  if (h->cfg.kind != GAST_KIND_MODEL) return fail("streaming is implemented for the MODEL kind only");
  if (!h->cfg.causal) return fail("streaming needs a causal model (gen_skes.py:59: causal=True): a non-causal network "
                                  "has no output for the newest frame");
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

extern "C" int gast_stream_push(gast_t* h, void* state, int64_t step, const float* x, float* y, int32_t n_streams,
                                const int32_t* fresh, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h) return fail("gast_stream_push: null handle");
  if (!h->prepared) return fail("gast_stream_push: gast_prepare() has not run since the last gast_bind()");
  if (step < 0 || !state || !x || !y) return fail("gast_stream_push: bad arguments");
  StreamPlan sp;
  if (stream_plan(h, n_streams, &sp)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUDA_OK(cudaSetDevice(h->cfg.device));
  if (!h->stream_ready && stream_prepare(h, st)) return 1;
  const size_t need = gast_stream_workspace_bytes(h, n_streams);
  if (!workspace || workspace_bytes < need)
    return fail("gast_stream_push: workspace too small (%zu < %zu bytes)", workspace_bytes, need);
  h->launches = 0; h->tc_launches = 0; h->ev_used = 0; h->ev_kind.clear();
  const gast_cfg& c = h->cfg;
  const int n = n_streams, J = c.num_joints, C = c.channels, L = c.num_stages, k0 = c.filter_widths[0], Fin = c.in_features;
  float* sbase = reinterpret_cast<float*>(align256(state));
  Arena a = workspace_arena(workspace, workspace_bytes);
  StreamBufs sb;
  stream_bufs(h, n, a, &sb);
  const long long rows = (long long)n * J;
  // input history + expand (gast_net.py:163-164) on the last k0 frames
  float* xhist = sbase + sp.xhist_off;
  stream_xpush_kernel<<<cdiv((long long)n * J * Fin, 256), 256, 0, st>>>(xhist, x, fresh, n, k0, J * Fin);
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
    const int p0 = hs % d, r = hs / d;
    const RowMap same{n, n, 1, 0};
    const ASeg taps = seg_taps(ring + (long long)p0 * slot_floats, Cw, Cw, fw, (long long)d * slot_floats, same);
    if (run_stage(h, st, s, n, taps, s.Wrot[r], &s.tc_rot[r], sb.tmp, ring + (long long)hs * slot_floats, same, sb.act))
      return 1;
    bout = (i < L - 1) ? slot_ptr(i + 1) : sb.fin;
    if (run_block(h, st, h->blocks[i], sb.act, n, sb.bb, bout)) return 1;
  }
  if (launch_shrink(h, st, bout, y, rows, nullptr, nullptr)) return 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}
