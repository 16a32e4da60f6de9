// Eval-mode backward and chunked eval-mode forward: a call covers its (clip, output frame) grid in passes of at most
// `max_frames` output positions, so its workspace depends on max_frames and the architecture, not on B or T; the
// unchunked eval backward is the one-pass plan (WHOLE_CALL).  A backward pass recomputes the activations from x with a
// frozen-BatchNorm training forward, then runs the training backward; nothing is held between the inference forward
// and the backward.  Included by gast_api.cu after train.cuh (uses its planning, sizing and training path).
//
// Under frozen BatchNorm every output position depends on its own receptive field only, so a pass is an ordinary
// call on a slice: whole clips when a clip's output fits a pass, else a window of output frames of one clip and the
// input frames that map to it.  Both are contiguous in x (B,T,J,F), y and dy (B,T_out,J,3), so a pass reads and
// writes them in place.  Gradients of the passes are summed in pass order (grad_add_multi_kernel); dL/dx of
// overlapping windows is added into place.
#pragma once

constexpr int GRAD_ADD_CHUNK = 4096;

// max_frames of the one-pass plan, which no public entry can pass: B * T_out may exceed INT32_MAX
constexpr long long WHOLE_CALL = LLONG_MAX;

static TrainState eval_state(int strided_now) {
  TrainState ts;
  ts.frozen = true; ts.sn = strided_now ? 1 : 0;
  return ts;
}

// dst[i] += src[i] over every chunk of a table of 3 int64 per chunk: {dst ptr, src ptr, count <= GRAD_ADD_CHUNK}.
// One block per chunk, so all parameter gradients of a pass are added in one launch.
__global__ void grad_add_multi_kernel(const long long* __restrict__ table) {
  const long long* e = table + 3LL * blockIdx.x;
  float* d = reinterpret_cast<float*>(e[0]);
  const float* s = reinterpret_cast<const float*>(e[1]);
  const int cnt = (int)e[2];
  for (int i = threadIdx.x; i < cnt; i += blockDim.x) d[i] += s[i];
}

// The pass plan of a call of B clips of T frames: the one rule the forward and the backward share.
//   T_out <= max_frames: a pass covers `clips` = min(B, max_frames / T_out) whole clips.
//   otherwise every clip is covered by windows of K = max_frames output frames (the last may be shorter); the
//   window of output frames [t0, t0 + k) reads input frames [t0 * S, t0 * S + (k - 1) * S + rf), S the output stride
//   of the schedule (1 dilated or dense, the product of the filter widths strided) and rf the receptive field.
// Passes run clip by clip, window by window; every output position falls in exactly one.
struct ChunkPlan {
  int T_out = 0, S = 1, rf = 1;
  bool windows = false;
  int clips = 1;              // whole clips per pass (!windows)
  int K = 0, wpc = 1;         // output frames per window and windows per clip (windows)
  long long passes = 0;
};

struct ChunkPass {
  int b0 = 0, nb = 0;         // clips [b0, b0 + nb)
  int t0 = 0, k = 0;          // their output frames [t0, t0 + k)
  int f0 = 0, Tin = 0;        // and the input frames [f0, f0 + Tin) those read
};

static ChunkPass chunk_pass(const ChunkPlan& pl, int B, int T, long long p) {
  ChunkPass q;
  if (!pl.windows) {
    q.b0 = (int)(p * pl.clips);
    q.nb = std::min(pl.clips, B - q.b0);
    q.k = pl.T_out; q.Tin = T;
    return q;
  }
  q.b0 = (int)(p / pl.wpc); q.nb = 1;
  q.t0 = (int)(p % pl.wpc) * pl.K;
  q.k = std::min(pl.K, pl.T_out - q.t0);
  q.f0 = q.t0 * pl.S;
  q.Tin = (q.k - 1) * pl.S + pl.rf;
  return q;
}

static int chunk_plan(const gast_handle* h, const char* who, int B, int T, int strided_now, long long max_frames,
                      ChunkPlan* pl) {
  if (h->cfg.kind != GAST_KIND_MODEL) return fail("%s: only the MODEL kind is chunked", who);
  if (max_frames < 1) return fail("%s: max_frames must be at least 1 (got %lld)", who, max_frames);
  if (B <= 0 || T <= 0) return fail("%s: empty batch (B=%d T=%d)", who, B, T);
  Geometry g;
  if (geometry(h, T, strided_now, &g)) return 1;
  pl->T_out = g.T_out;
  pl->S = g.s0;
  for (const StageGeo& s : g.stages) pl->S *= s.stride;
  pl->rf = gast_receptive_field(h);
  pl->windows = g.T_out > max_frames;
  if (!pl->windows) {
    pl->clips = (int)std::min<long long>(B, max_frames / g.T_out);
    pl->passes = ((long long)B + pl->clips - 1) / pl->clips;
  } else {
    pl->K = (int)max_frames;
    pl->wpc = (int)((g.T_out + max_frames - 1) / max_frames);
    pl->passes = (long long)B * pl->wpc;
  }
  // a window is an ordinary call whose output is exactly its k frames: check the full and the last one
  for (long long p : {0LL, pl->wpc - 1LL}) {
    const ChunkPass q = chunk_pass(*pl, B, T, p);
    if (q.f0 + q.Tin > T || gast_out_frames(h, q.Tin, strided_now) != q.k)
      return fail("%s: internal: window of %d input frames does not give %d outputs", who, q.Tin, q.k);
  }
  return 0;
}

// the largest pass of the plan: (clips, input frames)
static void chunk_full(const ChunkPlan& pl, int T, int* nb, int* Tin) {
  *nb = pl.windows ? 1 : pl.clips;
  *Tin = pl.windows ? (pl.K - 1) * pl.S + pl.rf : T;
}

// The backward's own area at the start of the workspace, taken by a plan of several passes only: the chunk table and a
// pass-gradient buffer per gradient tensor (with parameter gradients), and one window's dL/dx (windows).
struct ChunkArea {
  long long* table = nullptr;
  int n_chunks = 0;
  std::vector<float*> pass_grad;
  float* dxw = nullptr;
};

static void chunk_area(Arena& a, const std::vector<std::pair<std::string, int64_t>>& asked, const ChunkPlan& pl,
                       int T, int Fin_J, ChunkArea* ca) {
  if (pl.passes == 1) return;               // no area (a plan with windows has two passes at least)
  ca->n_chunks = 0;
  for (const auto& k : asked) ca->n_chunks += (int)((k.second + GRAD_ADD_CHUNK - 1) / GRAD_ADD_CHUNK);
  ca->table = reinterpret_cast<long long*>(a.take((size_t)6 * ca->n_chunks));
  ca->pass_grad.clear();
  for (const auto& k : asked) ca->pass_grad.push_back(a.take((size_t)k.second));
  int nb, Tin;
  chunk_full(pl, T, &nb, &Tin);
  if (pl.windows) ca->dxw = a.take((size_t)Tin * Fin_J);
}

// Workspace of an eval backward, by the sizing pass of its largest pass; 0 on error.  With several passes `asked`
// receives the gradient buffers that pass looks up; `dry` keeps its lookups for the caller to refuse on.
static size_t chunked_backward_sizing(gast_handle* h, TCtx& dry, int B, int T, int strided_now, const ChunkPlan& pl,
                                      std::vector<std::pair<std::string, int64_t>>* asked) {
  int nb, Tin;
  chunk_full(pl, T, &nb, &Tin);
  if (pl.passes > 1) dry.grad_bufs.asked = asked;
  const size_t pass = train_sizing(dry, nb, Tin, eval_state(strided_now));
  if (pass == 0) return 0;
  Arena a = sizing_arena();
  ChunkArea ca;
  chunk_area(a, *asked, pl, T, h->cfg.num_joints * h->cfg.in_features, &ca);
  return a.off + pass;
}

// The workspace query of an eval backward with parameter gradients, planned with `max_frames`: 0 when refused
static size_t eval_backward_workspace(gast_handle* h, const char* who, int B, int T, int strided_now,
                                      long long max_frames) {
  ChunkPlan pl;
  if (!h || train_check(h, who) || chunk_plan(h, who, B, T, strided_now, max_frames, &pl)) return 0;
  TCtx dry(h, nullptr, sizing_arena(), true);
  std::vector<std::pair<std::string, int64_t>> asked;
  return chunked_backward_sizing(h, dry, B, T, strided_now, pl, &asked);
}

extern "C" size_t gast_eval_backward_workspace_bytes(gast_t* h, int32_t B, int32_t T, int32_t strided_now) {
  return eval_backward_workspace(h, "gast_eval_backward_workspace_bytes", B, T, strided_now, WHOLE_CALL);
}

extern "C" size_t gast_chunked_workspace_bytes(gast_t* h, int32_t B, int32_t T, int32_t strided_now, int32_t max_frames,
                                               int32_t with_backward) {
  if (with_backward) return eval_backward_workspace(h, "gast_chunked_workspace_bytes", B, T, strided_now, max_frames);
  ChunkPlan pl;
  if (!h || chunk_plan(h, "gast_chunked_workspace_bytes", B, T, strided_now, max_frames, &pl)) return 0;
  int nb, Tin;
  chunk_full(pl, T, &nb, &Tin);
  return gast_workspace_bytes(h, nb, Tin, strided_now);
}

extern "C" int gast_forward_chunked(gast_t* h, const float* x, float* y, int32_t B, int32_t T, int32_t strided_now,
                                    int32_t max_frames, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h) return fail("gast_forward_chunked: null handle");
  if (!h->prepared) return fail("gast_forward_chunked: gast_prepare() has not run since the last gast_bind()");
  if (!x || !y) return fail("gast_forward_chunked: x and y must be device pointers");
  ChunkPlan pl;
  if (chunk_plan(h, "gast_forward_chunked", B, T, strided_now, max_frames, &pl)) return 1;
  int nb, Tin;
  chunk_full(pl, T, &nb, &Tin);
  const size_t need = gast_workspace_bytes(h, nb, Tin, strided_now);
  if (need == 0) return 1;
  if (call_begin(h, "gast_forward_chunked", need, workspace, workspace_bytes)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long xrow = (long long)h->cfg.num_joints * h->cfg.in_features, yrow = (long long)h->cfg.num_joints * 3;
  const size_t es = with_types(h, [](auto io, auto) { return sizeof(typename decltype(io)::type); });   // of x and y
  for (long long p = 0; p < pl.passes; ++p) {
    const ChunkPass q = chunk_pass(pl, B, T, p);
    const char* xp = reinterpret_cast<const char*>(x) + ((long long)q.b0 * T + q.f0) * xrow * es;
    char* yp = reinterpret_cast<char*>(y) + ((long long)q.b0 * pl.T_out + q.t0) * yrow * es;
    if (model_forward(h, st, reinterpret_cast<const float*>(xp), reinterpret_cast<float*>(yp), q.nb, q.Tin, strided_now,
                      workspace_arena(workspace, workspace_bytes), nullptr, nullptr))
      return 1;
  }
  return 0;
}

static int eval_backward(gast_handle* h, const char* who, const float* x, const float* dy, float* dx, int param_grads,
                         int B, int T, int strided_now, long long max_frames, void* workspace, size_t workspace_bytes,
                         void* stream) {
  if (!h) return fail("%s: null handle", who);
  if (train_check(h, who)) return 1;
  if (!x || !dy) return fail("%s: x and dy must be device pointers", who);
  if (!dx && !param_grads) return fail("%s: neither dx nor parameter gradients requested", who);
  ChunkPlan pl;
  if (chunk_plan(h, who, B, T, strided_now, max_frames, &pl)) return 1;
  const bool pgrad = param_grads != 0;
  TCtx dry(h, nullptr, sizing_arena(), pgrad);
  std::vector<std::pair<std::string, int64_t>> asked;
  const size_t need = chunked_backward_sizing(h, dry, B, T, strided_now, pl, &asked);
  if (need == 0 || dry.refuse(true)) return 1;
  if (call_begin(h, who, need, workspace, workspace_bytes)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int J = h->cfg.num_joints;
  const long long xrow = (long long)J * h->cfg.in_features, yrow = (long long)J * 3;
  Arena a = workspace_arena(workspace, workspace_bytes);
  ChunkArea ca;
  chunk_area(a, asked, pl, T, (int)xrow, &ca);
  const size_t pass_off = a.off;
  // the passes after the first write their parameter gradients into the pass-gradient area, which is then added to
  // the bound buffers the first pass wrote
  std::unordered_map<std::string, Binding> pass_bufs;
  if (pgrad && pl.passes > 1) {
    std::vector<long long> tab;
    for (size_t i = 0; i < asked.size(); ++i) {
      const int64_t n = asked[i].second;
      pass_bufs[asked[i].first] = Binding{ca.pass_grad[i], n};
      float* dst = reinterpret_cast<float*>(h->grads.at(asked[i].first).ptr);
      for (int64_t o = 0; o < n; o += GRAD_ADD_CHUNK)
        tab.insert(tab.end(), {(long long)(uintptr_t)(dst + o), (long long)(uintptr_t)(ca.pass_grad[i] + o),
                               (long long)std::min<int64_t>(GRAD_ADD_CHUNK, n - o)});
    }
    CUDA_OK(cudaMemcpyAsync(ca.table, tab.data(), tab.size() * sizeof(long long), cudaMemcpyHostToDevice, st));
  }
  // windows overlap by rf - 1 input frames: dL/dx starts at zero and every window adds its own
  if (dx && pl.windows) CUDA_OK(cudaMemsetAsync(dx, 0, sizeof(float) * (size_t)B * T * xrow, st));
  for (long long p = 0; p < pl.passes; ++p) {
    const ChunkPass q = chunk_pass(pl, B, T, p);
    const long long xoff = ((long long)q.b0 * T + q.f0) * xrow;
    float* dxp = !dx ? nullptr : pl.windows ? ca.dxw : dx + xoff;
    TCtx c(h, st, workspace_arena(workspace, workspace_bytes, pass_off), pgrad, p == 0 ? nullptr : &pass_bufs);
    TrainState ts = eval_state(strided_now);
    if (train_forward(h, c, ts, x + xoff, nullptr, q.nb, q.Tin)) return 1;
    c.tc_slot = 1024;
    if (train_backward(h, c, ts, dy + ((long long)q.b0 * pl.T_out + q.t0) * yrow, dxp)) return 1;
    if (dx && pl.windows) {
      const long long n = (long long)q.Tin * xrow;
      add_inplace_kernel<<<cdiv(n, 256), 256, 0, st>>>(dx + xoff, ca.dxw, n);
      h->launches++;
    }
    if (pgrad && p > 0) {
      grad_add_multi_kernel<<<ca.n_chunks, 256, 0, st>>>(ca.table);
      h->launches++;
    }
  }
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_eval_backward(gast_t* h, const float* x, const float* dy, float* dx, int32_t param_grads, int32_t B,
                                  int32_t T, int32_t strided_now, void* workspace, size_t workspace_bytes, void* stream) {
  return eval_backward(h, "gast_eval_backward", x, dy, dx, param_grads, B, T, strided_now, WHOLE_CALL, workspace,
                       workspace_bytes, stream);
}

extern "C" int gast_eval_backward_chunked(gast_t* h, const float* x, const float* dy, float* dx, int32_t param_grads,
                                          int32_t B, int32_t T, int32_t strided_now, int32_t max_frames, void* workspace,
                                          size_t workspace_bytes, void* stream) {
  return eval_backward(h, "gast_eval_backward_chunked", x, dy, dx, param_grads, B, T, strided_now, max_frames,
                       workspace, workspace_bytes, stream);
}
