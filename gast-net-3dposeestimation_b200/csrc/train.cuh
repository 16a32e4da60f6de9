// Training-mode forward and backward of the lifting network (SURVEY.md §8 row a12):
// SpatioTemporalModelOptimized1f in train() mode as main.train() uses it (main.py:213-243):
// batch-statistics BatchNorm with running-stat updates, Dropout, and the full backward down to
// every parameter of the reference's state_dict.  Included by gast_api.cu (uses its helpers).
//
// Everything a backward needs is kept in the caller's workspace (bump allocation, no reuse except the one partials
// area of the column reductions, col_reduce_area): the training batch is small (b=128 -> 19,584 / 6,528 / 2,176 rows),
// so memory is not the constraint.  No sum depends on the order in which blocks run: the tap adjoints are gathers
// (seg_adjoint_kernel) and the column sums are finished by their consumer in a fixed order (col_partials, col_total),
// so every call repeats bit for bit.
// Dense contractions run on the FFMA GEMM kernel (exact fp32); the frame-mapped operands of the
// temporal stages are gathered exactly as in inference.  Both schedules train: the strided one of
// SpatioTemporalModelOptimized1f (main.py:166-170) and the dilated one of SpatioTemporalModel (main.py:171-175).
// The same forward in frozen mode (TrainState::frozen: BatchNorm on the running statistics, no dropout, the inference
// schedule) recomputes the activations for the eval-mode backward; the backward also writes dL/dx, and skips every
// parameter-gradient kernel when only dL/dx is wanted (TCtx::pgrad).
//
// Every function here runs in two passes of one TCtx.  The sizing pass (an arena without memory) walks the same code
// as the launch pass and enqueues nothing: its arena takes give the workspace size, and it makes every parameter and
// gradient-buffer lookup the launch pass makes.  A failed lookup is recorded there, and each call refuses on that
// record (TCtx::refuse) before its first launch.
#pragma once

// ---------------------------------------------------------------------------------------------
struct TCtx {
  gast_handle* h; cudaStream_t st; Arena a; int J;
  bool dry;      // sizing pass: arena takes and lookups only, nothing is enqueued
  // backward: false = input gradient only (every parameter frozen): no weight-gradient contraction, no parameter-
  // gradient kernel, and no gradient buffer has to be bound
  bool pgrad;
  int tc_slot = 0;   // next slot of the handle's table of per-GEMM tensor-core operand copies (train_tcw)
  // the partials area of the column reductions (TrainState::red_part), set by train_forward and train_backward; the
  // reductions and their consumers run in stream order and share it
  double* red_part = nullptr;
  Lookup params, grad_bufs;
  // grads: where the gradient buffers are looked up, the handle's gast_bind_grads bindings unless given (the chunked
  // eval backward points the passes after its first at its pass-gradient area)
  TCtx(gast_handle* h_, cudaStream_t st_, Arena a_, bool pgrad_,
       const std::unordered_map<std::string, Binding>* grads = nullptr)
      : h(h_), st(st_), a(a_), J(h_->cfg.num_joints), dry(a_.dry), pgrad(pgrad_), params(h_),
        grad_bufs(grads ? Lookup(*grads, "gradient buffer") : Lookup(h_, true)) {}
  float* fl(size_t n) { return a.take(n); }
  double* dbl(size_t n) { return reinterpret_cast<double*>(a.take(2 * n)); }
  unsigned char* bytes(size_t n) { return reinterpret_cast<unsigned char*>(a.take((n + 3) / 4)); }
  float* param(const std::string& key, int64_t numel) { return params.get(key, numel); }
  // the gradient buffer bound for `key`, null when no parameter gradient is computed
  float* grad(const std::string& key, int64_t numel) { return pgrad ? grad_bufs.get(key, numel) : nullptr; }
  // nonzero with the error set when a lookup of this context failed: a parameter, or with grads a gradient buffer
  int refuse(bool grads) const {
    if (!params.ok) return fail("%s", params.err.c_str());
    if (grads && !grad_bufs.ok) return fail("%s", grad_bufs.err.c_str());
    return 0;
  }
  template <class... KP, class... A>
  void launch(void (*kernel)(KP...), dim3 grid, dim3 block, size_t smem, A&&... args) {
    if (!dry) kernel<<<grid, block, smem, st>>>(std::forward<A>(args)...);
  }
  void zero(void* p, size_t n) { if (!dry) cudaMemsetAsync(p, 0, n, st); }
  void copy(void* dst, const void* src, size_t n) {
    if (!dry) cudaMemcpyAsync(dst, src, n, cudaMemcpyDeviceToDevice, st);
  }
  // f() in the launch pass only: the counted launches of the inference code
  template <class F> int live(F f) { return dry ? 0 : f(); }
  // grid of a column reduction over M rows and N columns (col_partials); its consumer takes cdiv(N, 32) blocks
  static dim3 col_grid(long long M, int N) {
    return dim3(cdiv(N, 32), (unsigned)std::min<long long>(COL_RED_ROWS, (M + 7) / 8));
  }
};

// The column reductions' partials area of a training forward of B clips of T frames and of its backward: the widest
// reduction has max(in_features, the last block's 2 x channels) columns, and none has more rows than init_bn's B*T*J.
static void col_reduce_area(TCtx& c, TrainState& ts, int B, int T) {
  const gast_cfg& cf = c.h->cfg;
  const int N = std::max({cf.in_features, cf.channels << cf.num_stages, 8});
  const long long R = TCtx::col_grid((long long)B * T * c.J, N).y;
  ts.red_part = c.dbl((size_t)R * 2 * N);
  c.red_part = ts.red_part;
}

// dX = the adjoint of the tap gather `sg` of F output frames (seg_adjoint_kernel): sg.base is dX, its taps are
// sg.tap_stride / (J * sg.ld) frames apart, src holds the gathered gradient (row stride lds); plus the residual slice
// of map rmap from rsrc (row stride ldr) when rsrc is given.  Writes every element of dX.
static void seg_adjoint(TCtx& c, const ASeg& sg, long long F, const float* src, int lds, RowMap rmap = RowMap{1, 1, 1, 0},
                        const float* rsrc = nullptr, int ldr = 0) {
  const int taps = sg.K / sg.Kc;
  const int dil = (int)(sg.tap_stride / ((long long)c.J * sg.ld));
  const long long F_in = F / sg.map.T_out * sg.map.T_in;
  c.launch(seg_adjoint_kernel, cdiv(F_in * c.J * sg.Kc, 256), 256, 0, sg.map, taps, dil, sg.Kc, src, lds, rmap, rsrc,
           ldr, c.J, F_in, const_cast<float*>(sg.base), sg.ld);
}

// Tensor-core operand copies of one training GEMM's weight matrix (forward: the raw weights, backward: their transposes):
// the weights change every step, so the hi/lo split runs per call; buffers live in a per-handle table indexed by the
// GEMM's position in the step (the sequence of GEMMs of a model is fixed).  3xTF32 arithmetic (gemm_tc.cuh; inference
// runs the equally precise F16X3 form), the arithmetic the gradient-noise bars of tests/test_gpu_train.py were set
// against; one TF32 product in the TF32 training precision (launch_gemm picks it from h->train_precision).  Shapes
// the core does not take (K % 16: the expand conv) stay on FFMA.
static const TcWeights* train_tcw(TCtx& c, const float* W, int N, int K) {
  const size_t slot = (size_t)c.tc_slot++;
  if (c.h->gemm_core != 0) return nullptr;
  if (c.h->train_tc.size() <= slot) c.h->train_tc.resize(slot + 1);
  TcWeights& t = c.h->train_tc[slot];
  if (tc_prepare_weights(t, W, N, K, c.st, &c.h->owned, false)) return nullptr;
  return t.ready ? &t : nullptr;
}

// dense out[M][N] = A[M][K] . W[N][K]^T (+bias), rows are plain (no frame structure)
static int dense_nt(TCtx& c, const float* A, int lda, const float* W, long long M, int N, int K, float* out, int ldo,
                    const float* bias = nullptr) {
  if (M <= 0) return 0;
  GemmP p;
  gemm_flat(p, M);
  p.nseg = 1; p.seg[0] = seg_flat(A, lda, K);
  p.W = W; p.ldw = K; p.N = N; p.out = out; p.ld_out = ldo; p.bias = bias;
  return c.live([&] { return launch_gemm(c.h, c.st, EPI_PLAIN, p, train_tcw(c, W, N, K)); });
}

// frame-structured forward GEMM with gathered segments (same kernel as inference), raw weights
static int seg_gemm(TCtx& c, const ASeg* segs, int nseg, const float* W, int ldw, long long F, int N, float* out,
                    int ldo, const float* bias = nullptr) {
  if (F <= 0) return 0;
  GemmP p;
  gemm_defaults(p, c.h, F);
  p.nseg = nseg;
  for (int i = 0; i < nseg; ++i) p.seg[i] = segs[i];
  p.W = W; p.ldw = ldw; p.N = N; p.out = out; p.ld_out = ldo; p.bias = bias;
  return c.live([&] { return launch_gemm(c.h, c.st, EPI_PLAIN, p, train_tcw(c, W, N, ldw)); });
}

static long long pad32(long long m) { return (m + 31) / 32 * 32; }

// row splits *S of *rps rows each of the weight-gradient contraction over M rows: enough CTAs for two waves of the
// machine, at least 256 rows per split
static void wgrad_split(long long M, int N, int K, int sm_count, long long* S, long long* rps) {
  const int tiles = (int)(cdiv(N, WG_T) * cdiv(K, WG_T));
  long long s = std::max<long long>(1, std::min<long long>((M + 255) / 256, (2LL * sm_count + tiles - 1) / tiles));
  const long long r = ((M + s - 1) / s + WG_M - 1) / WG_M * WG_M;
  s = r > 0 ? (M + r - 1) / r : 1;
  *S = s < 1 ? 1 : s;
  *rps = r;
}

// the split contraction into part (S * N * K floats) and the fixed-order reduction of the partials into dW.  tf32:
// wgrad_tc_kernel where it takes the shape (*on_tc = true), wgrad_tn_kernel (exact fp32) otherwise.  0 or a cudaError_t.
static int wgrad_run(cudaStream_t st, const float* dZ, int lddz, const float* A, int lda, long long M, int N, int K,
                     long long S, long long rps, float* part, float* dW, int lddw, bool tf32, bool* on_tc) {
  *on_tc = tf32 && wgrad_tc_takes(dZ, lddz, N, K);
  if (*on_tc) {
    const int rc = wgrad_tc_launch(st, dZ, lddz, A, lda, M, N, K, rps, S, part);
    if (rc) return rc;
  } else {
    dim3 grid(cdiv(N, WG_T), cdiv(K, WG_T), (unsigned)S);
    wgrad_tn_kernel<<<grid, 256, 0, st>>>(dZ, lddz, A, lda, M, N, K, rps, part);
  }
  wgrad_reduce_kernel<<<cdiv((long long)N * K, 256), 256, 0, st>>>(part, (int)S, N, K, dW, lddw);
  return (int)cudaGetLastError();
}

// dW[N][K] = dZ[M][N]^T . A[M][K]: split over the rows + fixed-order reduction of the partials (wgrad_run); on the
// TF32 tensor-core kernel in the TF32 training precision on the tensor-core core
static int dense_tn(TCtx& c, const float* dZ, int lddz, const float* A, int lda, long long M, int N, int K, float* dW,
                    int lddw) {
  if (!c.pgrad) return 0;   // every use is a parameter gradient
  long long S, rps;
  wgrad_split(M, N, K, c.h->sm_count, &S, &rps);
  float* part = c.fl((size_t)S * N * K);
  if (M <= 0) return 0;
  return c.live([&] {
    bool on_tc = false;
    const int rc = wgrad_run(c.st, dZ, lddz, A, lda, M, N, K, S, rps, part, dW, lddw,
                             c.h->gemm_core == 0 && c.h->train_precision == 1, &on_tc);
    if (rc) return fail("weight-gradient launch failed: %s", cudaGetErrorString((cudaError_t)rc));
    c.h->launches += 2;
    if (on_tc) c.h->wgrad_tc_launches++;
    return 0;
  });
}

// dA[M][K] = dZ[M][N] . W[N][K]   (W transposed on the fly)
static int dense_nn(TCtx& c, const float* dZ, int lddz, const float* W, int ldw, long long M, int N, int K, float* dA,
                    int ldda) {
  const int Np = (int)pad32(N);
  float* Wt = c.fl((size_t)K * Np);
  c.zero(Wt, sizeof(float) * (size_t)K * Np);
  c.launch(transpose_kernel, dim3(cdiv(N, 32), cdiv(K, 32)), dim3(32, 8), 0, W, N, K, ldw, Wt, Np);
  if (Np == N) return dense_nt(c, dZ, lddz, Wt, M, K, Np, dA, ldda);
  float* dZp = c.fl((size_t)M * Np);
  c.zero(dZp, sizeof(float) * (size_t)M * Np);
  c.launch(copy2d_kernel, cdiv(M * N, 256), 256, 0, dZ, lddz, dZp, Np, M, N, 0);
  return dense_nt(c, dZp, Np, Wt, M, K, Np, dA, ldda);
}

// backward of the 1x1 conv Z[M][N] = A[M][K] . W^T whose weight W[N][K] is bound as `key`: its weight gradient into
// the gradient buffer of `key` (c.pgrad), then dA = dZ . W
static int conv1x1_bwd(TCtx& c, const std::string& key, const float* dZ, const float* A, long long M, int N, int K,
                       float* dA) {
  if (dense_tn(c, dZ, N, A, K, M, N, K, c.grad(key, (int64_t)N * K), K)) return 1;
  return dense_nn(c, dZ, N, c.param(key, (int64_t)N * K), K, M, N, K, dA, K);
}

// ---- BatchNorm, training mode (batch statistics) or frozen (running statistics: ts.frozen) ----------------
static int bn_fwd(TCtx& c, BnSave& s, const std::string& prefix, const float* Z, int ldz, long long M, int N, int relu,
                  float drop_p, TrainState& ts, const float* res, int ldres, RowMap rmap, float* Y, int ldy) {
  s.prefix = prefix; s.Z = Z; s.ldz = ldz; s.M = M; s.N = N; s.relu = relu; s.frozen = ts.frozen;
  s.mean = c.fl(N); s.invstd = c.fl(N);
  if (ts.frozen) drop_p = 0.f;   // eval semantics whatever the module's dropout
  unsigned char* keep = nullptr;
  s.kscale = 1.f;
  if (drop_p > 0.f) { keep = c.bytes((size_t)M * N); s.kscale = 1.f / (1.f - drop_p); }
  s.keep = keep;
  s.gamma = c.param(prefix + "weight", N); s.beta = c.param(prefix + "bias", N);
  float* rm = c.param(prefix + "running_mean", N);
  float* rv = c.param(prefix + "running_var", N);
  if (ts.frozen) {
    c.launch(bn_running_kernel, cdiv(N, 128), 128, 0, rm, rv, N, s.mean, s.invstd);
  } else {
    const dim3 grid = TCtx::col_grid(M, N);
    c.launch(col_stats_kernel, grid, 256, 0, Z, M, N, ldz, c.red_part);
    c.launch(bn_finalize_kernel, grid.x, 256, 0, c.red_part, (int)grid.y, M, N, s.mean, s.invstd, rm, rv, 0.1f);
  }
  if (keep) {
    const unsigned long long seed = ts.seed + 0x51ED270B * (++ts.drop_ctr);
    c.launch(dropout_mask_kernel, cdiv(M * N, 256), 256, 0, keep, M * N, drop_p, seed, c.h->dropout_state);
  }
  c.launch(bn_apply_kernel, cdiv(M * N, 256), 256, 0, Z, ldz, s.mean, s.invstd, s.gamma, s.beta, relu, res, ldres, rmap,
           c.J, keep, s.kscale, Y, ldy, M, N);
  return 0;
}

// dZ from dY; writes the weight/bias gradients of this BatchNorm (c.pgrad).  The column sums dgamma = sum dY'.xhat,
// dbeta = sum dY' are those gradients; batch statistics also need them for dZ, running statistics do not.
static int bn_bwd(TCtx& c, const BnSave& s, const float* dY, int lddy, float* dZ, int lddz) {
  double* sums = (!s.frozen || c.pgrad) ? c.dbl(2 * (size_t)s.N) : nullptr;
  float* gw = c.grad(s.prefix + "weight", s.N);
  float* gb = c.grad(s.prefix + "bias", s.N);
  if (sums) {
    const dim3 grid = TCtx::col_grid(s.M, s.N);
    c.launch(bn_bwd_reduce_kernel, grid, 256, 0, dY, lddy, s.Z, s.ldz, s.mean, s.invstd, s.gamma, s.beta, s.relu,
             s.keep, s.kscale, s.M, s.N, c.red_part);
    c.launch(col_total_kernel<2>, grid.x, 256, 0, c.red_part, (int)grid.y, s.N, sums, nullptr);
  }
  const double* dg = sums;
  const double* db = sums ? sums + s.N : nullptr;
  c.launch(s.frozen ? bn_bwd_apply_kernel<true> : bn_bwd_apply_kernel<false>, cdiv(s.M * s.N, 256), 256, 0, dY, lddy,
           s.Z, s.ldz, s.mean, s.invstd, s.gamma, s.beta, s.relu, s.keep, s.kscale, s.M, s.N, dg, db, dZ, lddz, gw, gb);
  return 0;
}

static NbrRows nbr_rows(const NbrTable& nb, int J) {
  NbrRows r;
  memset(&r, 0, sizeof(r));
  for (int i = 0; i < J; ++i)
    for (int z = nb.row_ptr[i]; z < nb.row_ptr[i + 1]; ++z) r.rowof[z] = (unsigned char)i;
  return r;
}

// ---- GraphAttentionBlock, training forward ---------------------------------------------------------
static int block_fwd(TCtx& c, TrainState& ts, BlockSave& b, BlockConsts& bc, const std::string& P, const float* X,
                     long long F) {
  gast_handle* h = c.h;
  const int C = bc.C, J = c.J;
  const long long M = F * J;
  b.C = C; b.F = F; b.X = X; b.P = P;
  const std::string lp = P + "local_graph_layer.", gp = P + "global_graph_layer.";
  const RowMap id{1, 1, 1, 0};
  b.Wst = c.fl((size_t)4 * C * C);
  b.H = c.fl((size_t)M * 4 * C);
  b.coefA[0] = c.fl((size_t)h->nnz[0] * C); b.coefA[1] = c.fl((size_t)h->nnz[1] * C);
  b.S = c.fl((size_t)M * 2 * C); b.XY = c.fl((size_t)M * 2 * C);
  b.Zlc = c.fl((size_t)M * C); b.L = c.fl((size_t)M * C);
  b.G = c.fl((size_t)M * C); b.AB = c.fl((size_t)M * 8); b.Y = c.fl((size_t)M * C);
  b.Zgc = c.fl((size_t)M * C); b.Gl = c.fl((size_t)M * C);
  b.Zbc = c.fl((size_t)M * 2 * C); b.Out = c.fl((size_t)M * 2 * C);
  // ---- local
  for (int m = 0; m < 2; ++m) {
    const std::string g = lp + (m == 0 ? "gcn_sym." : "gcn_con.");
    const float* W = c.param(g + "W", (int64_t)2 * C * C);
    const float* e = c.param(g + "e", (int64_t)C * h->nnz[m]);
    c.launch(semch_wstack_kernel, cdiv((long long)2 * C * C, 256), 256, 0, W, C, C, b.Wst + (size_t)m * 2 * C * C);
    BnP none{nullptr, nullptr, nullptr, nullptr};
    c.launch(semch_coef_kernel, cdiv((long long)C * J, 128), 128, 0, b.coefA[m], nullptr, e, h->nnz[m], h->nbr[m],
             h->nnz[m], C, J, none, nullptr);
  }
  if (dense_nt(c, X, C, b.Wst, M, 4 * C, C, b.H, 4 * C)) return 1;
  for (int m = 0; m < 2; ++m)
    c.launch(semch_mix_fwd_kernel, cdiv(M * C, 256), 256, 0, b.H + m * 2 * C, 4 * C, b.coefA[m], h->nbr[m], J, F, C,
             b.S + m * C, 2 * C);
  if (bn_fwd(c, b.bn1, lp + "bn_1.", b.S, 2 * C, M, C, 1, 0.f, ts, nullptr, 0, id, b.XY, 2 * C)) return 1;
  if (bn_fwd(c, b.bn2, lp + "bn_2.", b.S + C, 2 * C, M, C, 1, 0.f, ts, nullptr, 0, id, b.XY + C, 2 * C)) return 1;
  if (dense_nt(c, b.XY, 2 * C, c.param(lp + "cat_conv.weight", (int64_t)C * 2 * C), M, C, 2 * C, b.Zlc, C)) return 1;
  if (bn_fwd(c, b.bnlc, lp + "cat_bn.", b.Zlc, C, M, C, 1, ts.drop_p, ts, nullptr, 0, id, b.L, C)) return 1;
  // ---- global (stacked g / collapsed theta,phi constants are refreshed here, they follow the weights)
  GlobalParams gpar;
  global_params(h, c.params, bc, gp, GAST_KIND_MGLOBAL, &gpar);
  if (c.live([&] { return prepare_global(h, c.st, bc, gpar, GAST_KIND_MGLOBAL); })) return 1;
  if (dense_nt(c, X, C, bc.Wg, M, C, C, b.G, C, bc.bg)) return 1;
  if (c.live([&] { return launch_rowdot(h, c.st, Elem<float>(), X, C, bc, b.AB, M); })) return 1;
  c.launch(att_mix_fwd_kernel, (unsigned)F, 256, sizeof(float) * 4 * J * J, b.G, C, b.AB, bc.Ck, J, 4, C / 4, b.Y, C);
  if (dense_nt(c, b.Y, C, c.param(gp + "cat_conv.weight", (int64_t)C * C), M, C, C, b.Zgc, C)) return 1;
  if (bn_fwd(c, b.bngc, gp + "cat_bn.", b.Zgc, C, M, C, 1, ts.drop_p, ts, nullptr, 0, id, b.Gl, C)) return 1;
  // ---- cat[x, local, global] -> 1x1 -> BN -> ReLU
  const ASeg segs[3] = {seg_flat(X, C, C), seg_flat(b.L, C, C), seg_flat(b.Gl, C, C)};
  if (seg_gemm(c, segs, 3, c.param(P + "cat_conv.weight", (int64_t)2 * C * 3 * C), 3 * C, F, 2 * C, b.Zbc, 2 * C))
    return 1;
  if (bn_fwd(c, b.bnbc, P + "cat_bn.", b.Zbc, 2 * C, M, 2 * C, 1, 0.f, ts, nullptr, 0, id, b.Out, 2 * C)) return 1;
  return 0;
}

// ---- GraphAttentionBlock, backward: dOut (M x 2C) -> dX (M x C, overwritten) ----------------------------
// att_mix_bwd_kernel keeps four 4 x J x J tables in dynamic shared memory, 16 J^2 floats: 50,176 B at J = 28 and
// 65,536 B at J = 32 (gast_create's limit), over the 48 KB a launch gets without opting in.  The opt-in is per device.
static int att_mix_bwd_optin(const gast_handle* h) {
  static bool done[64];
  bool& d = done[h->cfg.device & 63];
  if (!d) {
    CUDA_OK(cudaFuncSetAttribute((const void*)att_mix_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)sizeof(float) * 16 * 32 * 32));
    d = true;
  }
  return 0;
}

static int block_bwd(TCtx& c, const BlockSave& b, BlockConsts& bc, const float* dOut, float* dX) {
  gast_handle* h = c.h;
  const int C = b.C, J = c.J;
  const long long F = b.F, M = F * J;
  const std::string& P = b.P;
  const std::string lp = P + "local_graph_layer.", gp = P + "global_graph_layer.";
  // (a) block cat
  float* dZbc = c.fl((size_t)M * 2 * C);
  if (bn_bwd(c, b.bnbc, dOut, 2 * C, dZbc, 2 * C)) return 1;
  float* Acat = c.fl((size_t)M * 3 * C);
  float* dAcat = c.fl((size_t)M * 3 * C);
  if (c.pgrad) {
    c.launch(copy2d_kernel, cdiv(M * C, 256), 256, 0, b.X, C, Acat, 3 * C, M, C, 0);
    c.launch(copy2d_kernel, cdiv(M * C, 256), 256, 0, b.L, C, Acat + C, 3 * C, M, C, 0);
    c.launch(copy2d_kernel, cdiv(M * C, 256), 256, 0, b.Gl, C, Acat + 2 * C, 3 * C, M, C, 0);
  }
  if (conv1x1_bwd(c, P + "cat_conv.weight", dZbc, Acat, M, 2 * C, 3 * C, dAcat)) return 1;
  c.launch(copy2d_kernel, cdiv(M * C, 256), 256, 0, dAcat, 3 * C, dX, C, M, C, 0);
  // (b) global branch
  float* dZgc = c.fl((size_t)M * C);
  if (bn_bwd(c, b.bngc, dAcat + 2 * C, 3 * C, dZgc, C)) return 1;
  float* dY = c.fl((size_t)M * C);
  if (conv1x1_bwd(c, gp + "cat_conv.weight", dZgc, b.Y, M, C, C, dY)) return 1;
  float* dG = c.fl((size_t)M * C);
  float* dab = c.fl((size_t)M * 8);
  float* dCk = c.fl((size_t)4 * J * J);
  float* dCkp = c.fl((size_t)F * 4 * J * J);     // per-frame contributions, reduced in a fixed order
  float* dWg = c.fl((size_t)C * C);
  float* dU = c.fl((size_t)8 * C);
  float* dbg = c.fl(C);
  float* dcab = c.fl(8);
  float* dXg = c.fl((size_t)M * C);
  if (c.live([&] { return att_mix_bwd_optin(h); })) return 1;
  c.launch(att_mix_bwd_kernel, (unsigned)F, 256, sizeof(float) * 16 * J * J, dY, C, b.G, C, b.AB, bc.Ck, J, 4, C / 4,
           dG, C, dab, dCkp);
  if (c.live([&] {
        const cudaError_t e = cudaGetLastError();
        return e == cudaSuccess ? 0 : fail("att_mix_bwd_kernel launch failed (J=%d): %s", J, cudaGetErrorString(e));
      }))
    return 1;
  if (c.pgrad) {
    c.launch(col_sum_det_kernel, cdiv(4 * J * J, 32), 256, 0, dCkp, F, 4 * J * J, dCk);
    const dim3 g1 = TCtx::col_grid(M, C), g2 = TCtx::col_grid(M, 8);
    c.launch(col_sum_kernel, g1, 256, 0, dG, M, C, C, c.red_part);
    c.launch(col_total_kernel<1>, g1.x, 256, 0, c.red_part, (int)g1.y, C, nullptr, dbg);
    c.launch(col_sum_kernel, g2, 256, 0, dab, M, 8, 8, c.red_part);
    c.launch(col_total_kernel<1>, g2.x, 256, 0, c.red_part, (int)g2.y, 8, nullptr, dcab);
  }
  if (dense_tn(c, dG, C, b.X, C, M, C, C, dWg, C)) return 1;
  if (dense_nn(c, dG, C, bc.Wg, C, M, C, C, dXg, C)) return 1;
  // dU[8][C] = dab[M][8]^T . X[M][C]: the same row-contraction as a weight gradient (a one-thread-per-output
  // kernel took 3.4 ms per block at b = 128)
  if (dense_tn(c, dab, 8, b.X, C, M, 8, C, dU, C)) return 1;
  c.launch(rowdot_bwd_x_kernel, cdiv(M * C, 256), 256, 0, dab, bc.U, 8, M, C, dXg, C);
  c.launch(add_inplace_kernel, cdiv(M * C, 256), 256, 0, dX, dXg, M * C);
  const int Cg = C / 4;
  for (int hd = 0; hd < (c.pgrad ? 4 : 0); ++hd) {
    const std::string hp = gp + "attentions." + std::to_string(hd) + ".";
    c.copy(c.grad(hp + "g.weight", (int64_t)Cg * C), dWg + (size_t)hd * Cg * C, sizeof(float) * Cg * C);
    c.copy(c.grad(hp + "g.bias", Cg), dbg + hd * Cg, sizeof(float) * Cg);
    c.copy(c.grad(hp + "C_k", (int64_t)J * J), dCk + hd * J * J, sizeof(float) * J * J);
    const float* tw = c.param(hp + "theta.weight", (int64_t)Cg * C);
    const float* tb = c.param(hp + "theta.bias", Cg);
    const float* pw = c.param(hp + "phi.weight", (int64_t)Cg * C);
    const float* pb = c.param(hp + "phi.bias", Cg);
    const float* wc = c.param(hp + "concat_project.0.weight", 2 * Cg);
    float* gtw = c.grad(hp + "theta.weight", (int64_t)Cg * C);
    float* gtb = c.grad(hp + "theta.bias", Cg);
    float* gpw = c.grad(hp + "phi.weight", (int64_t)Cg * C);
    float* gpb = c.grad(hp + "phi.bias", Cg);
    float* gwc = c.grad(hp + "concat_project.0.weight", 2 * Cg);
    c.launch(global_collapse_bwd_kernel, Cg, 128, 0, dU, dcab, hd, C, Cg, tw, tb, pw, pb, wc, gtw, gtb, gpw, gpb, gwc);
  }
  // (c) local branch
  float* dZlc = c.fl((size_t)M * C);
  if (bn_bwd(c, b.bnlc, dAcat + C, 3 * C, dZlc, C)) return 1;
  float* dXY = c.fl((size_t)M * 2 * C);
  if (conv1x1_bwd(c, lp + "cat_conv.weight", dZlc, b.XY, M, C, 2 * C, dXY)) return 1;
  float* dS = c.fl((size_t)M * 2 * C);
  if (bn_bwd(c, b.bn1, dXY, 2 * C, dS, 2 * C)) return 1;
  if (bn_bwd(c, b.bn2, dXY + C, 2 * C, dS + C, 2 * C)) return 1;
  float* dH = c.fl((size_t)M * 4 * C);
  float* dWst = c.fl((size_t)4 * C * C);
  float* dXl = c.fl((size_t)M * C);
  for (int m = 0; m < 2; ++m) {
    float* dA = c.fl((size_t)h->nnz[m] * C);
    const int dsplit = (int)std::max<long long>(1, std::min<long long>(32, F / 32));   // frame ranges of semch_dcoef_kernel
    double* dpart = c.dbl((size_t)dsplit * h->nnz[m] * C);
    float* ge = c.grad(lp + (m == 0 ? "gcn_sym.e" : "gcn_con.e"), (int64_t)C * h->nnz[m]);
    const NbrRows nr = nbr_rows(h->nbr[m], J);
    c.launch(semch_mix_bwd_kernel, cdiv(M * C, 256), 256, 0, dS + m * C, 2 * C, b.coefA[m], h->nbr[m], nr, h->nnz[m], J,
             F, C, dH + m * 2 * C, 4 * C);
    if (!c.pgrad) continue;
    c.launch(semch_dcoef_kernel, dim3(cdiv((long long)h->nnz[m] * C, 128), dsplit), 128, 0, dS + m * C, 2 * C,
             b.H + m * 2 * C, 4 * C, h->nbr[m], nr, h->nnz[m], J, F, C, dpart);
    c.launch(semch_dcoef_reduce_kernel, cdiv((long long)h->nnz[m] * C, 128), 128, 0, dpart, dsplit, h->nnz[m] * C, dA);
    c.launch(semch_de_kernel, cdiv((long long)C * J, 128), 128, 0, b.coefA[m], dA, h->nbr[m], h->nnz[m], J, C, ge);
  }
  if (dense_tn(c, dH, 4 * C, b.X, C, M, 4 * C, C, dWst, C)) return 1;
  if (dense_nn(c, dH, 4 * C, b.Wst, C, M, 4 * C, C, dXl, C)) return 1;
  c.launch(add_inplace_kernel, cdiv(M * C, 256), 256, 0, dX, dXl, M * C);
  for (int m = 0; m < (c.pgrad ? 2 : 0); ++m)
    c.launch(semch_wgrad_relayout_kernel, cdiv((long long)2 * C * C, 256), 256, 0, dWst + (size_t)m * 2 * C * C, C, C,
             C, c.grad(lp + (m == 0 ? "gcn_sym.W" : "gcn_con.W"), (int64_t)2 * C * C));
  return 0;
}

// ---- whole model ---------------------------------------------------------------------------------
// y may be null (the eval backward recomputes the activations only)
static int train_forward(gast_handle* h, TCtx& c, TrainState& ts, const float* x, float* y, int B, int T) {
  const gast_cfg& cf = h->cfg;
  const int J = c.J, C = cf.channels, L = cf.num_stages, Fin = cf.in_features, k0 = cf.filter_widths[0];
  // schedule = the handle's own: strided for SpatioTemporalModelOptimized1f (main.py:166-170), dilated (or the
  // dense ablation) for SpatioTemporalModel (main.py:171-175, `--disable-optimizations` / stride > 1).  Batch
  // statistics are taken over every position the reference computes, so a dilated model never runs the
  // needed-only schedule in training.  Frozen BatchNorm makes the positions independent: the eval-mode forward
  // takes the schedule gast_forward takes (ts.sn), and a dilated model fed one receptive field computes only
  // the positions its output needs.
  const int sn = ts.frozen ? ts.sn : (cf.strided ? 1 : 0);
  if (geometry(h, T, sn, &ts.geo)) return 1;
  const Geometry& g = ts.geo;
  ts.B = B; ts.T = T; ts.x = x;
  ts.blocks.assign(L, BlockSave());
  ts.stages.assign(L - 1, StageSave());
  const RowMap id{1, 1, 1, 0};
  // expand: init_bn (batch stats over every input position) -> conv(k0, stride k0) -> BN -> ReLU
  const long long Min = (long long)B * T * J, F0 = (long long)B * g.T0, M0 = F0 * J;
  const int KP = (k0 * Fin + 7) / 8 * 8;
  ts.xbn = c.fl((size_t)Min * Fin);
  ts.Acol = c.fl((size_t)M0 * KP);
  ts.We8 = c.fl((size_t)C * KP);
  ts.Z0 = c.fl((size_t)M0 * C);
  ts.act0 = c.fl((size_t)M0 * C);
  col_reduce_area(c, ts, B, T);
  if (bn_fwd(c, ts.bnin, "init_bn.", x, Fin, Min, Fin, 0, 0.f, ts, nullptr, 0, id, ts.xbn, Fin)) return 1;
  const float* we = c.param("expand_conv.weight", (int64_t)C * Fin * k0);
  float* tmp = c.fl((size_t)C * k0 * Fin);
  c.zero(ts.Acol, sizeof(float) * (size_t)M0 * KP);
  c.zero(ts.We8, sizeof(float) * (size_t)C * KP);
  const ASeg sg = seg_taps(ts.xbn, Fin, Fin, k0, (long long)J * Fin, RowMap{g.T0, T, g.s0, 0});
  c.launch(seg_gather_kernel, cdiv(M0 * sg.K, 256), 256, 0, sg, J, F0, ts.Acol, KP, 0);
  BnP none{nullptr, nullptr, nullptr, nullptr};
  // We8[c][tap*Fin + i] = w[c][i][tap]  (fold_conv_kernel with no BN is exactly this re-layout)
  c.launch(fold_conv_kernel, cdiv((long long)C * Fin * k0, 256), 256, 0, tmp, nullptr, we, C, Fin, k0, none);
  c.launch(copy2d_kernel, cdiv((long long)C * k0 * Fin, 256), 256, 0, tmp, k0 * Fin, ts.We8, KP, C, k0 * Fin, 0);
  if (dense_nt(c, ts.Acol, KP, ts.We8, M0, C, KP, ts.Z0, C)) return 1;
  if (bn_fwd(c, ts.bnex, "expand_bn.", ts.Z0, C, M0, C, 1, 0.f, ts, nullptr, 0, id, ts.act0, C)) return 1;
  if (block_fwd(c, ts, ts.blocks[0], h->blocks[0], "layers_graph_conv.0.", ts.act0, F0)) return 1;
  const float* cur = ts.blocks[0].Out;
  for (int i = 1; i < L; ++i) {
    StageSave& s = ts.stages[i - 1];
    const StageGeo& sgeo = g.stages[i - 1];
    const int Cw = C << i;
    const long long Fn = (long long)B * sgeo.Tout, Mn = Fn * J;
    s.g = sgeo; s.Cw = Cw; s.X = cur; s.idx = i - 1;
    s.Wt = c.fl((size_t)Cw * sgeo.taps * Cw);
    s.Z1 = c.fl((size_t)Mn * Cw); s.Hh = c.fl((size_t)Mn * Cw); s.Z2 = c.fl((size_t)Mn * Cw); s.Out = c.fl((size_t)Mn * Cw);
    const float* w0 = c.param("layers_conv." + std::to_string(2 * (i - 1)) + ".weight", (int64_t)Cw * Cw * sgeo.taps);
    const float* w1 = c.param("layers_conv." + std::to_string(2 * (i - 1) + 1) + ".weight", (int64_t)Cw * Cw);
    c.launch(fold_conv_kernel, cdiv((long long)Cw * Cw * sgeo.taps, 256), 256, 0, s.Wt, nullptr, w0, Cw, Cw, sgeo.taps,
             none);
    const ASeg taps = seg_taps(cur, Cw, Cw, sgeo.taps, (long long)sgeo.dil * J * Cw, sgeo.tapmap);
    if (seg_gemm(c, &taps, 1, s.Wt, sgeo.taps * Cw, Fn, Cw, s.Z1, Cw)) return 1;
    if (bn_fwd(c, s.bnA, "layers_bn." + std::to_string(2 * (i - 1)) + ".", s.Z1, Cw, Mn, Cw, 1, 0.f, ts, nullptr, 0, id,
               s.Hh, Cw)) return 1;
    if (dense_nt(c, s.Hh, Cw, w1, Mn, Cw, Cw, s.Z2, Cw)) return 1;
    if (bn_fwd(c, s.bnB, "layers_bn." + std::to_string(2 * (i - 1) + 1) + ".", s.Z2, Cw, Mn, Cw, 1, ts.drop_p, ts, cur, Cw,
               sgeo.resmap, s.Out, Cw)) return 1;
    if (block_fwd(c, ts, ts.blocks[i], h->blocks[i], "layers_graph_conv." + std::to_string(i) + ".", s.Out, Fn)) return 1;
    cur = ts.blocks[i].Out;
  }
  ts.last = cur;
  const int Cl = C << L;
  const long long M = (long long)B * g.T_out * J;
  const float* ws = c.param("shrink.weight", (int64_t)3 * Cl);
  if (y) c.launch(shrink_kernel<float, float>, cdiv(M * 32, 256), 256, 0, cur, Cl, ws, y, M, Cl);
  return 0;
}

// dy -> the parameter gradients (c.pgrad) and dL/dx into dx (B,T,J,F; may be null)
static int train_backward(gast_handle* h, TCtx& c, const TrainState& ts, const float* dy, float* dx) {
  const gast_cfg& cf = h->cfg;
  const int J = c.J, C = cf.channels, L = cf.num_stages, Fin = cf.in_features, k0 = cf.filter_widths[0];
  const int Cl = C << L;
  const Geometry& g = ts.geo;
  c.red_part = ts.red_part;
  // shrink
  const long long M = (long long)ts.B * g.T_out * J;
  float* dcur = c.fl((size_t)M * Cl);
  const float* ws = c.param("shrink.weight", (int64_t)3 * Cl);
  float* gws = c.grad("shrink.weight", (int64_t)3 * Cl);
  c.launch(shrink_bwd_x_kernel, cdiv(M * Cl, 256), 256, 0, dy, ws, M, Cl, dcur);
  if (gws) c.launch(shrink_bwd_w_kernel, cdiv(Cl, 32), dim3(32, SBW_RG), 0, dy, ts.last, M, Cl, gws);
  for (int i = L - 1; i >= 1; --i) {
    const StageSave& s = ts.stages[i - 1];
    const int Cw = s.Cw, taps = s.g.taps;
    const long long Fout = (long long)ts.B * s.g.Tout, Mn = Fout * J, Mi = (long long)ts.B * s.g.Tin * J;
    float* dSout = c.fl((size_t)Mn * Cw);
    if (block_bwd(c, ts.blocks[i], h->blocks[i], dcur, dSout)) return 1;
    // stage: out = res + drop(relu(bn(conv1x1(h))));  h = relu(bn(conv_taps(x)))
    float* dXin = c.fl((size_t)Mi * Cw);
    float* dZ2 = c.fl((size_t)Mn * Cw);
    float* dHh = c.fl((size_t)Mn * Cw);
    float* dZ1 = c.fl((size_t)Mn * Cw);
    float* Xcol = c.fl((size_t)Mn * taps * Cw);
    float* dXcol = c.fl((size_t)Mn * taps * Cw);
    float* dWt = c.fl((size_t)Cw * taps * Cw);
    if (bn_bwd(c, s.bnB, dSout, Cw, dZ2, Cw)) return 1;
    if (conv1x1_bwd(c, "layers_conv." + std::to_string(2 * s.idx + 1) + ".weight", dZ2, s.Hh, Mn, Cw, Cw, dHh)) return 1;
    if (bn_bwd(c, s.bnA, dHh, Cw, dZ1, Cw)) return 1;
    const ASeg sg = seg_taps(s.X, Cw, Cw, taps, (long long)s.g.dil * J * Cw, s.g.tapmap);
    if (c.pgrad) c.launch(seg_gather_kernel, cdiv(Mn * sg.K, 256), 256, 0, sg, J, Fout, Xcol, taps * Cw, 0);
    if (dense_tn(c, dZ1, Cw, Xcol, taps * Cw, Mn, Cw, taps * Cw, dWt, taps * Cw)) return 1;
    if (dense_nn(c, dZ1, Cw, s.Wt, taps * Cw, Mn, Cw, taps * Cw, dXcol, taps * Cw)) return 1;
    float* gw0 = c.grad("layers_conv." + std::to_string(2 * s.idx) + ".weight", (int64_t)Cw * Cw * taps);
    if (gw0)
      c.launch(conv_wgrad_relayout_kernel, cdiv((long long)Cw * Cw * taps, 256), 256, 0, dWt, Cw, Cw, taps, taps * Cw, gw0);
    // dXin = the residual slice's gradient, then the taps' (one fixed order, every element written once)
    ASeg dsg = sg; dsg.base = dXin;
    seg_adjoint(c, dsg, Fout, dXcol, taps * Cw, s.g.resmap, dSout, Cw);
    dcur = dXin;
  }
  // first block
  const long long F0 = (long long)ts.B * g.T0, M0 = F0 * J;
  float* dAct0 = c.fl((size_t)M0 * C);
  if (block_bwd(c, ts.blocks[0], h->blocks[0], dcur, dAct0)) return 1;
  // expand
  const int KP = (k0 * Fin + 7) / 8 * 8;
  const long long Min = (long long)ts.B * ts.T * J;
  float* dZ0 = c.fl((size_t)M0 * C);
  if (bn_bwd(c, ts.bnex, dAct0, C, dZ0, C)) return 1;
  float* dWe8 = c.fl((size_t)C * KP);
  float* dAcol = c.fl((size_t)M0 * KP);
  float* dxbn = c.fl((size_t)Min * Fin);
  float* dxin = c.fl((size_t)Min * Fin);
  if (dense_tn(c, dZ0, C, ts.Acol, KP, M0, C, KP, dWe8, KP)) return 1;
  if (dense_nn(c, dZ0, C, ts.We8, KP, M0, C, KP, dAcol, KP)) return 1;
  float* gwe = c.grad("expand_conv.weight", (int64_t)C * Fin * k0);
  if (gwe) c.launch(conv_wgrad_relayout_kernel, cdiv((long long)C * Fin * k0, 256), 256, 0, dWe8, C, Fin, k0, KP, gwe);
  const ASeg sg = seg_taps(dxbn, Fin, Fin, k0, (long long)J * Fin, RowMap{g.T0, ts.T, g.s0, 0});
  seg_adjoint(c, sg, F0, dAcol, KP);
  // init_bn: dx = dxbn . gamma . invstd (frozen), the batch-statistics adjoint otherwise
  if (bn_bwd(c, ts.bnin, dxbn, Fin, dx ? dx : dxin, Fin)) return 1;
  return 0;
}
