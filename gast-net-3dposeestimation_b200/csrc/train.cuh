// Training-mode forward and backward of the lifting network (SURVEY.md §8 row a12):
// SpatioTemporalModelOptimized1f in train() mode as main.train() uses it (main.py:213-243):
// batch-statistics BatchNorm with running-stat updates, Dropout, and the full backward down to
// every parameter of the reference's state_dict.  Included by gast_api.cu (uses its helpers).
//
// Everything a backward needs is kept in the caller's workspace (bump allocation, no reuse): the
// training batch is small (b=128 -> 19,584 / 6,528 / 2,176 rows), so memory is not the constraint.
// Dense contractions run on the FFMA GEMM kernel (exact fp32); the frame-mapped operands of the
// temporal stages are gathered exactly as in inference.  Both schedules train: the strided one of
// SpatioTemporalModelOptimized1f (main.py:166-170) and the dilated one of SpatioTemporalModel (main.py:171-175).
// The same forward in frozen mode (TrainState::frozen: BatchNorm on the running statistics, no dropout, the inference
// schedule) recomputes the activations for the eval-mode backward; the backward also writes dL/dx, and skips every
// parameter-gradient kernel when only dL/dx is wanted (TCtx::pgrad).
#pragma once

// ---------------------------------------------------------------------------------------------
struct TCtx {
  gast_handle* h; cudaStream_t st; Arena* a; Lookup* L; int J;
  bool dry;   // sizing pass: no launches
  int tc_slot = 0;   // next slot of the handle's table of per-GEMM tensor-core operand copies (train_tcw)
  // backward: false = input gradient only (every parameter frozen): no weight-gradient contraction, no parameter-
  // gradient kernel, and no gradient buffer has to be bound
  bool pgrad = true;
  float* fl(size_t n) { return a->take(n); }
  double* dbl(size_t n) { return reinterpret_cast<double*>(a->take(2 * n)); }
  unsigned char* bytes(size_t n) { return reinterpret_cast<unsigned char*>(a->take((n + 3) / 4)); }
};

static float* grad_ptr(gast_handle* h, const std::string& key, int64_t numel) {
  auto it = h->grads.find(key);
  if (it == h->grads.end()) { fail("gradient buffer for '%s' is not bound", key.c_str()); return nullptr; }
  if (it->second.numel != numel) { fail("gradient buffer '%s' has the wrong size", key.c_str()); return nullptr; }
  return reinterpret_cast<float*>(it->second.ptr);
}

// *out = the bound gradient buffer of `key`, or null when no parameter gradient is computed (sizing pass, input-only
// backward).  false: a wanted buffer is missing or has the wrong size.
static bool want_grad(TCtx& c, const std::string& key, int64_t numel, float** out) {
  *out = nullptr;
  if (c.dry || !c.pgrad) return true;
  *out = grad_ptr(c.h, key, numel);
  return *out != nullptr;
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
  if (c.dry || M <= 0) return 0;
  GemmP p;
  gemm_flat(p, M);
  p.nseg = 1; p.seg[0] = seg_flat(A, lda, K);
  p.W = W; p.ldw = K; p.N = N; p.out = out; p.ld_out = ldo; p.bias = bias;
  return launch_gemm(c.h, c.st, EPI_PLAIN, p, train_tcw(c, W, N, K));
}

// frame-structured forward GEMM with gathered segments (same kernel as inference), raw weights
static int seg_gemm(TCtx& c, const ASeg* segs, int nseg, const float* W, int ldw, long long F, int N, float* out,
                    int ldo, const float* bias = nullptr) {
  if (c.dry || F <= 0) return 0;
  GemmP p;
  gemm_defaults(p, c.h, F);
  p.nseg = nseg;
  for (int i = 0; i < nseg; ++i) p.seg[i] = segs[i];
  p.W = W; p.ldw = ldw; p.N = N; p.out = out; p.ld_out = ldo; p.bias = bias;
  return launch_gemm(c.h, c.st, EPI_PLAIN, p, train_tcw(c, W, N, ldw));
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
  if (c.dry || M <= 0) return 0;
  bool on_tc = false;
  const int rc = wgrad_run(c.st, dZ, lddz, A, lda, M, N, K, S, rps, part, dW, lddw,
                           c.h->gemm_core == 0 && c.h->train_precision == 1, &on_tc);
  if (rc) return fail("weight-gradient launch failed: %s", cudaGetErrorString((cudaError_t)rc));
  c.h->launches += 2;
  if (on_tc) c.h->wgrad_tc_launches++;
  return 0;
}

// dA[M][K] = dZ[M][N] . W[N][K]   (W transposed on the fly)
static int dense_nn(TCtx& c, const float* dZ, int lddz, const float* W, int ldw, long long M, int N, int K, float* dA,
                    int ldda) {
  const int Np = (int)pad32(N);
  float* Wt = c.fl((size_t)K * Np);
  float* dZp = nullptr;
  if (Np != N) dZp = c.fl((size_t)M * Np);
  if (c.dry) return 0;
  cudaMemsetAsync(Wt, 0, sizeof(float) * (size_t)K * Np, c.st);
  transpose_kernel<<<dim3(cdiv(N, 32), cdiv(K, 32)), dim3(32, 8), 0, c.st>>>(W, N, K, ldw, Wt, Np);
  const float* dz = dZ; int ld = lddz;
  if (dZp) {
    cudaMemsetAsync(dZp, 0, sizeof(float) * (size_t)M * Np, c.st);
    copy2d_kernel<<<cdiv(M * N, 256), 256, 0, c.st>>>(dZ, lddz, dZp, Np, M, N, 0);
    dz = dZp; ld = Np;
  }
  return dense_nt(c, dz, ld, Wt, M, K, Np, dA, ldda);
}

// ---- BatchNorm, training mode (batch statistics) or frozen (running statistics: ts.frozen) ----------------
static int bn_fwd(TCtx& c, BnSave& s, const std::string& prefix, const float* Z, int ldz, long long M, int N, int relu,
                  float drop_p, TrainState& ts, const float* res, int ldres, RowMap rmap, float* Y, int ldy) {
  s.prefix = prefix; s.Z = Z; s.ldz = ldz; s.M = M; s.N = N; s.relu = relu; s.frozen = ts.frozen;
  s.mean = c.fl(N); s.invstd = c.fl(N);
  double* sums = ts.frozen ? nullptr : c.dbl(2 * (size_t)N);
  if (ts.frozen) drop_p = 0.f;   // eval semantics whatever the module's dropout
  unsigned char* keep = nullptr;
  s.kscale = 1.f;
  if (drop_p > 0.f) { keep = c.bytes((size_t)M * N); s.kscale = 1.f / (1.f - drop_p); }
  s.keep = keep;
  if (c.dry) return 0;
  s.gamma = c.L->get(prefix + "weight", N); s.beta = c.L->get(prefix + "bias", N);
  float* rm = const_cast<float*>(c.L->get(prefix + "running_mean", N));
  float* rv = const_cast<float*>(c.L->get(prefix + "running_var", N));
  if (!c.L->ok) return 1;
  if (ts.frozen) {
    bn_running_kernel<<<cdiv(N, 128), 128, 0, c.st>>>(rm, rv, N, s.mean, s.invstd);
  } else {
    cudaMemsetAsync(sums, 0, sizeof(double) * 2 * N, c.st);
    dim3 grid(cdiv(N, 32), (unsigned)std::min<long long>(256, (M + 7) / 8));
    col_stats_kernel<<<grid, 256, 0, c.st>>>(Z, M, N, ldz, sums, sums + N);
    bn_finalize_kernel<<<cdiv(N, 128), 128, 0, c.st>>>(sums, sums + N, M, N, s.mean, s.invstd, rm, rv, 0.1f);
  }
  if (keep) {
    dropout_mask_kernel<<<cdiv(M * N, 256), 256, 0, c.st>>>(keep, M * N, drop_p, ts.seed + 0x51ED270B * (++ts.drop_ctr), c.h->dropout_state);
  }
  bn_apply_kernel<<<cdiv(M * N, 256), 256, 0, c.st>>>(Z, ldz, s.mean, s.invstd, s.gamma, s.beta, relu, res, ldres, rmap,
                                                    c.J, keep, s.kscale, Y, ldy, M, N);
  return 0;
}

// dZ from dY; writes the weight/bias gradients of this BatchNorm (c.pgrad).  The column sums dgamma = sum dY'.xhat,
// dbeta = sum dY' are those gradients; batch statistics also need them for dZ, running statistics do not.
static int bn_bwd(TCtx& c, const BnSave& s, const float* dY, int lddy, float* dZ, int lddz) {
  double* sums = (!s.frozen || c.pgrad) ? c.dbl(2 * (size_t)s.N) : nullptr;
  float *gw, *gb;
  if (!want_grad(c, s.prefix + "weight", s.N, &gw) || !want_grad(c, s.prefix + "bias", s.N, &gb)) return 1;
  if (c.dry) return 0;
  if (sums) {
    cudaMemsetAsync(sums, 0, sizeof(double) * 2 * s.N, c.st);
    dim3 grid(cdiv(s.N, 32), (unsigned)std::min<long long>(256, (s.M + 7) / 8));
    bn_bwd_reduce_kernel<<<grid, 256, 0, c.st>>>(dY, lddy, s.Z, s.ldz, s.mean, s.invstd, s.gamma, s.beta, s.relu, s.keep,
                                                s.kscale, s.M, s.N, sums, sums + s.N);
  }
  const double* dg = sums;
  const double* db = sums ? sums + s.N : nullptr;
  if (s.frozen)
    bn_bwd_apply_kernel<true><<<cdiv(s.M * s.N, 256), 256, 0, c.st>>>(dY, lddy, s.Z, s.ldz, s.mean, s.invstd, s.gamma,
                                                                      s.beta, s.relu, s.keep, s.kscale, s.M, s.N, dg, db,
                                                                      dZ, lddz, gw, gb);
  else
    bn_bwd_apply_kernel<false><<<cdiv(s.M * s.N, 256), 256, 0, c.st>>>(dY, lddy, s.Z, s.ldz, s.mean, s.invstd, s.gamma,
                                                                       s.beta, s.relu, s.keep, s.kscale, s.M, s.N, dg, db,
                                                                       dZ, lddz, gw, gb);
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
  if (!c.dry) {
    for (int m = 0; m < 2; ++m) {
      const std::string g = lp + (m == 0 ? "gcn_sym." : "gcn_con.");
      const float* W = c.L->get(g + "W", (int64_t)2 * C * C);
      const float* e = c.L->get(g + "e", (int64_t)C * h->nnz[m]);
      if (!c.L->ok) return 1;
      semch_wstack_kernel<<<cdiv((long long)2 * C * C, 256), 256, 0, c.st>>>(W, C, C, b.Wst + (size_t)m * 2 * C * C);
      BnP none{nullptr, nullptr, nullptr, nullptr};
      semch_coef_kernel<<<cdiv((long long)C * J, 128), 128, 0, c.st>>>(b.coefA[m], nullptr, e, h->nnz[m], h->nbr[m],
                                                                      h->nnz[m], C, J, none, nullptr);
    }
  }
  if (dense_nt(c, X, C, b.Wst, M, 4 * C, C, b.H, 4 * C)) return 1;
  if (!c.dry)
    for (int m = 0; m < 2; ++m)
      semch_mix_fwd_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(b.H + m * 2 * C, 4 * C, b.coefA[m], h->nbr[m], J, F, C,
                                                              b.S + m * C, 2 * C);
  if (bn_fwd(c, b.bn1, lp + "bn_1.", b.S, 2 * C, M, C, 1, 0.f, ts, nullptr, 0, id, b.XY, 2 * C)) return 1;
  if (bn_fwd(c, b.bn2, lp + "bn_2.", b.S + C, 2 * C, M, C, 1, 0.f, ts, nullptr, 0, id, b.XY + C, 2 * C)) return 1;
  {
    const float* w = c.dry ? nullptr : c.L->get(lp + "cat_conv.weight", (int64_t)C * 2 * C);
    if (!c.dry && !c.L->ok) return 1;
    if (dense_nt(c, b.XY, 2 * C, w, M, C, 2 * C, b.Zlc, C)) return 1;
  }
  if (bn_fwd(c, b.bnlc, lp + "cat_bn.", b.Zlc, C, M, C, 1, ts.drop_p, ts, nullptr, 0, id, b.L, C)) return 1;
  // ---- global (stacked g / collapsed theta,phi constants are refreshed here, they follow the weights)
  if (!c.dry) {
    if (prepare_global(h, *c.L, c.st, bc, gp, GAST_KIND_MGLOBAL)) return 1;
  }
  if (dense_nt(c, X, C, bc.Wg, M, C, C, b.G, C, bc.bg)) return 1;
  if (!c.dry) {
    if (launch_rowdot(h, c.st, X, C, bc, b.AB, M)) return 1;
    att_mix_fwd_kernel<<<(unsigned)F, 256, sizeof(float) * 4 * J * J, c.st>>>(b.G, C, b.AB, bc.Ck, J, 4, C / 4, b.Y, C);
  }
  {
    const float* w = c.dry ? nullptr : c.L->get(gp + "cat_conv.weight", (int64_t)C * C);
    if (!c.dry && !c.L->ok) return 1;
    if (dense_nt(c, b.Y, C, w, M, C, C, b.Zgc, C)) return 1;
  }
  if (bn_fwd(c, b.bngc, gp + "cat_bn.", b.Zgc, C, M, C, 1, ts.drop_p, ts, nullptr, 0, id, b.Gl, C)) return 1;
  // ---- cat[x, local, global] -> 1x1 -> BN -> ReLU
  {
    const float* w = c.dry ? nullptr : c.L->get(P + "cat_conv.weight", (int64_t)2 * C * 3 * C);
    if (!c.dry && !c.L->ok) return 1;
    ASeg segs[3] = {seg_flat(X, C, C), seg_flat(b.L, C, C), seg_flat(b.Gl, C, C)};
    if (seg_gemm(c, segs, 3, w, 3 * C, F, 2 * C, b.Zbc, 2 * C)) return 1;
  }
  if (bn_fwd(c, b.bnbc, P + "cat_bn.", b.Zbc, 2 * C, M, 2 * C, 1, 0.f, ts, nullptr, 0, id, b.Out, 2 * C)) return 1;
  return 0;
}

// ---- GraphAttentionBlock, backward: dOut (M x 2C) -> dX (M x C, overwritten) ----------------------------
static int block_bwd(TCtx& c, BlockSave& b, BlockConsts& bc, const float* dOut, float* dX) {
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
  if (!c.dry && c.pgrad) {
    copy2d_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(b.X, C, Acat, 3 * C, M, C, 0);
    copy2d_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(b.L, C, Acat + C, 3 * C, M, C, 0);
    copy2d_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(b.Gl, C, Acat + 2 * C, 3 * C, M, C, 0);
  }
  {
    const float* w = c.dry ? nullptr : c.L->get(P + "cat_conv.weight", (int64_t)2 * C * 3 * C);
    float* gw;
    if (!want_grad(c, P + "cat_conv.weight", (int64_t)2 * C * 3 * C, &gw) || (!c.dry && !c.L->ok)) return 1;
    if (dense_tn(c, dZbc, 2 * C, Acat, 3 * C, M, 2 * C, 3 * C, gw, 3 * C)) return 1;
    if (dense_nn(c, dZbc, 2 * C, w, 3 * C, M, 2 * C, 3 * C, dAcat, 3 * C)) return 1;
  }
  if (!c.dry) copy2d_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(dAcat, 3 * C, dX, C, M, C, 0);
  // (b) global branch
  float* dZgc = c.fl((size_t)M * C);
  if (bn_bwd(c, b.bngc, dAcat + 2 * C, 3 * C, dZgc, C)) return 1;
  float* dY = c.fl((size_t)M * C);
  {
    const float* w = c.dry ? nullptr : c.L->get(gp + "cat_conv.weight", (int64_t)C * C);
    float* gw;
    if (!want_grad(c, gp + "cat_conv.weight", (int64_t)C * C, &gw) || (!c.dry && !c.L->ok)) return 1;
    if (dense_tn(c, dZgc, C, b.Y, C, M, C, C, gw, C)) return 1;
    if (dense_nn(c, dZgc, C, w, C, M, C, C, dY, C)) return 1;
  }
  float* dG = c.fl((size_t)M * C);
  float* dab = c.fl((size_t)M * 8);
  float* dCk = c.fl((size_t)4 * J * J);
  float* dCkp = c.fl((size_t)F * 4 * J * J);     // per-frame contributions, reduced in a fixed order
  float* dWg = c.fl((size_t)C * C);
  float* dU = c.fl((size_t)8 * C);
  double* dsum = c.dbl((size_t)C + 8);
  float* dbg = c.fl(C);
  float* dcab = c.fl(8);
  float* dXg = c.fl((size_t)M * C);
  if (!c.dry) {
    att_mix_bwd_kernel<<<(unsigned)F, 256, sizeof(float) * 16 * J * J, c.st>>>(dY, C, b.G, C, b.AB, bc.Ck, J, 4, C / 4, dG,
                                                                               C, dab, dCkp);
    if (c.pgrad) {
      col_sum_det_kernel<<<cdiv(4 * J * J, 32), 256, 0, c.st>>>(dCkp, F, 4 * J * J, dCk);
      cudaMemsetAsync(dsum, 0, sizeof(double) * (C + 8), c.st);
      dim3 g1(cdiv(C, 32), (unsigned)std::min<long long>(256, (M + 7) / 8));
      col_sum_kernel<<<g1, 256, 0, c.st>>>(dG, M, C, C, dsum);
      dim3 g2(1, (unsigned)std::min<long long>(256, (M + 7) / 8));
      col_sum_kernel<<<g2, 256, 0, c.st>>>(dab, M, 8, 8, dsum + C);
      d2f_kernel<<<cdiv(C, 128), 128, 0, c.st>>>(dsum, dbg, C);
      d2f_kernel<<<1, 32, 0, c.st>>>(dsum + C, dcab, 8);
    }
  }
  if (dense_tn(c, dG, C, b.X, C, M, C, C, dWg, C)) return 1;
  if (dense_nn(c, dG, C, bc.Wg, C, M, C, C, dXg, C)) return 1;
  // dU[8][C] = dab[M][8]^T . X[M][C]: the same row-contraction as a weight gradient (a one-thread-per-output
  // kernel took 3.4 ms per block at b = 128)
  if (dense_tn(c, dab, 8, b.X, C, M, 8, C, dU, C)) return 1;
  if (!c.dry) {
    rowdot_bwd_x_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(dab, bc.U, 8, M, C, dXg, C);
    add_inplace_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(dX, dXg, M * C);
    const int Cg = C / 4;
    for (int hd = 0; hd < (c.pgrad ? 4 : 0); ++hd) {
      const std::string hp = gp + "attentions." + std::to_string(hd) + ".";
      float* ggw = grad_ptr(h, hp + "g.weight", (int64_t)Cg * C);
      float* ggb = grad_ptr(h, hp + "g.bias", Cg);
      float* gck = grad_ptr(h, hp + "C_k", (int64_t)J * J);
      float* gtw = grad_ptr(h, hp + "theta.weight", (int64_t)Cg * C);
      float* gtb = grad_ptr(h, hp + "theta.bias", Cg);
      float* gpw = grad_ptr(h, hp + "phi.weight", (int64_t)Cg * C);
      float* gpb = grad_ptr(h, hp + "phi.bias", Cg);
      float* gwc = grad_ptr(h, hp + "concat_project.0.weight", 2 * Cg);
      if (!ggw || !ggb || !gck || !gtw || !gtb || !gpw || !gpb || !gwc) return 1;
      cudaMemcpyAsync(ggw, dWg + (size_t)hd * Cg * C, sizeof(float) * Cg * C, cudaMemcpyDeviceToDevice, c.st);
      cudaMemcpyAsync(ggb, dbg + hd * Cg, sizeof(float) * Cg, cudaMemcpyDeviceToDevice, c.st);
      cudaMemcpyAsync(gck, dCk + hd * J * J, sizeof(float) * J * J, cudaMemcpyDeviceToDevice, c.st);
      const float* tw = c.L->get(hp + "theta.weight", (int64_t)Cg * C);
      const float* tb = c.L->get(hp + "theta.bias", Cg);
      const float* pw = c.L->get(hp + "phi.weight", (int64_t)Cg * C);
      const float* pb = c.L->get(hp + "phi.bias", Cg);
      const float* wc = c.L->get(hp + "concat_project.0.weight", 2 * Cg);
      if (!c.L->ok) return 1;
      global_collapse_bwd_kernel<<<Cg, 128, 0, c.st>>>(dU, dcab, hd, C, Cg, tw, tb, pw, pb, wc, gtw, gtb, gpw, gpb, gwc);
    }
  }
  // (c) local branch
  float* dZlc = c.fl((size_t)M * C);
  if (bn_bwd(c, b.bnlc, dAcat + C, 3 * C, dZlc, C)) return 1;
  float* dXY = c.fl((size_t)M * 2 * C);
  {
    const float* w = c.dry ? nullptr : c.L->get(lp + "cat_conv.weight", (int64_t)C * 2 * C);
    float* gw;
    if (!want_grad(c, lp + "cat_conv.weight", (int64_t)C * 2 * C, &gw) || (!c.dry && !c.L->ok)) return 1;
    if (dense_tn(c, dZlc, C, b.XY, 2 * C, M, C, 2 * C, gw, 2 * C)) return 1;
    if (dense_nn(c, dZlc, C, w, 2 * C, M, C, 2 * C, dXY, 2 * C)) return 1;
  }
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
    const std::string g = lp + (m == 0 ? "gcn_sym." : "gcn_con.");
    float* ge;
    if (!want_grad(c, g + "e", (int64_t)C * h->nnz[m], &ge)) return 1;
    if (c.dry) continue;
    NbrRows nr = nbr_rows(h->nbr[m], J);
    semch_mix_bwd_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(dS + m * C, 2 * C, b.coefA[m], h->nbr[m], nr, h->nnz[m], J, F,
                                                            C, dH + m * 2 * C, 4 * C);
    if (!c.pgrad) continue;
    semch_dcoef_kernel<<<dim3(cdiv((long long)h->nnz[m] * C, 128), dsplit), 128, 0, c.st>>>(
        dS + m * C, 2 * C, b.H + m * 2 * C, 4 * C, h->nbr[m], nr, h->nnz[m], J, F, C, dpart);
    semch_dcoef_reduce_kernel<<<cdiv((long long)h->nnz[m] * C, 128), 128, 0, c.st>>>(dpart, dsplit, h->nnz[m] * C, dA);
    semch_de_kernel<<<cdiv((long long)C * J, 128), 128, 0, c.st>>>(b.coefA[m], dA, h->nbr[m], h->nnz[m], J, C, ge);
  }
  if (dense_tn(c, dH, 4 * C, b.X, C, M, 4 * C, C, dWst, C)) return 1;
  if (dense_nn(c, dH, 4 * C, b.Wst, C, M, 4 * C, C, dXl, C)) return 1;
  if (!c.dry) {
    add_inplace_kernel<<<cdiv(M * C, 256), 256, 0, c.st>>>(dX, dXl, M * C);
    for (int m = 0; m < (c.pgrad ? 2 : 0); ++m) {
      const std::string g = lp + (m == 0 ? "gcn_sym." : "gcn_con.");
      float* gW = grad_ptr(h, g + "W", (int64_t)2 * C * C);
      if (!gW) return 1;
      semch_wgrad_relayout_kernel<<<cdiv((long long)2 * C * C, 256), 256, 0, c.st>>>(dWst + (size_t)m * 2 * C * C, C, C, C, gW);
    }
  }
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
  Geometry g;
  if (geometry(h, T, sn, &g)) return 1;
  ts.B = B; ts.T = T; ts.T0 = g.T0; ts.s0 = g.s0; ts.x = x;
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
  if (bn_fwd(c, ts.bnin, "init_bn.", x, Fin, Min, Fin, 0, 0.f, ts, nullptr, 0, id, ts.xbn, Fin)) return 1;
  if (!c.dry) {
    const float* we = c.L->get("expand_conv.weight", (int64_t)C * Fin * k0);
    if (!c.L->ok) return 1;
    cudaMemsetAsync(ts.Acol, 0, sizeof(float) * (size_t)M0 * KP, c.st);
    cudaMemsetAsync(ts.We8, 0, sizeof(float) * (size_t)C * KP, c.st);
    const ASeg sg = seg_taps(ts.xbn, Fin, Fin, k0, (long long)J * Fin, RowMap{g.T0, T, g.s0, 0});
    seg_gather_kernel<<<cdiv(M0 * sg.K, 256), 256, 0, c.st>>>(sg, J, F0, ts.Acol, KP, 0);
    BnP none{nullptr, nullptr, nullptr, nullptr};
    // We8[c][tap*Fin + i] = w[c][i][tap]  (fold_conv_kernel with no BN is exactly this re-layout)
    float* tmp = c.fl((size_t)C * k0 * Fin);
    fold_conv_kernel<<<cdiv((long long)C * Fin * k0, 256), 256, 0, c.st>>>(tmp, nullptr, we, C, Fin, k0, none);
    copy2d_kernel<<<cdiv((long long)C * k0 * Fin, 256), 256, 0, c.st>>>(tmp, k0 * Fin, ts.We8, KP, C, k0 * Fin, 0);
  } else {
    c.fl((size_t)C * k0 * Fin);
  }
  if (dense_nt(c, ts.Acol, KP, ts.We8, M0, C, KP, ts.Z0, C)) return 1;
  if (bn_fwd(c, ts.bnex, "expand_bn.", ts.Z0, C, M0, C, 1, 0.f, ts, nullptr, 0, id, ts.act0, C)) return 1;
  if (block_fwd(c, ts, ts.blocks[0], h->blocks[0], "layers_graph_conv.0.", ts.act0, F0)) return 1;
  const float* cur = ts.blocks[0].Out;
  long long F = F0;
  int Tp = g.T0;
  for (int i = 1; i < L; ++i) {
    StageSave& s = ts.stages[i - 1];
    Sched sc;
    stage_sched(h, i, sn, &sc);
    const int Cw = C << i, Tn = g.Ts[i - 1];
    const long long Fn = (long long)B * Tn, Mn = Fn * J;
    s.Cw = Cw; s.taps = sc.taps; s.Fin = F; s.Fout = Fn; s.Tin = Tp; s.Tout = Tn; s.X = cur; s.idx = i - 1; s.dil = sc.dil;
    s.tapmap = RowMap{Tn, Tp, sc.stride, 0};
    s.resmap = RowMap{Tn, Tp, sc.res_mul, sc.res_off};
    s.Wt = c.fl((size_t)Cw * sc.taps * Cw);
    s.Z1 = c.fl((size_t)Mn * Cw); s.Hh = c.fl((size_t)Mn * Cw); s.Z2 = c.fl((size_t)Mn * Cw); s.Out = c.fl((size_t)Mn * Cw);
    const std::string k0s = "layers_conv." + std::to_string(2 * (i - 1)) + ".weight";
    const std::string k1s = "layers_conv." + std::to_string(2 * (i - 1) + 1) + ".weight";
    const float* w1 = nullptr;
    if (!c.dry) {
      const float* w0 = c.L->get(k0s, (int64_t)Cw * Cw * sc.taps);
      w1 = c.L->get(k1s, (int64_t)Cw * Cw);
      if (!c.L->ok) return 1;
      BnP none{nullptr, nullptr, nullptr, nullptr};
      fold_conv_kernel<<<cdiv((long long)Cw * Cw * sc.taps, 256), 256, 0, c.st>>>(s.Wt, nullptr, w0, Cw, Cw, sc.taps, none);
    }
    const ASeg sg = seg_taps(cur, Cw, Cw, sc.taps, (long long)sc.dil * J * Cw, s.tapmap);
    if (seg_gemm(c, &sg, 1, s.Wt, sc.taps * Cw, Fn, Cw, s.Z1, Cw)) return 1;
    if (bn_fwd(c, s.bnA, "layers_bn." + std::to_string(2 * (i - 1)) + ".", s.Z1, Cw, Mn, Cw, 1, 0.f, ts, nullptr, 0, id,
               s.Hh, Cw)) return 1;
    if (dense_nt(c, s.Hh, Cw, w1, Mn, Cw, Cw, s.Z2, Cw)) return 1;
    if (bn_fwd(c, s.bnB, "layers_bn." + std::to_string(2 * (i - 1) + 1) + ".", s.Z2, Cw, Mn, Cw, 1, ts.drop_p, ts, cur, Cw,
               s.resmap, s.Out, Cw)) return 1;
    if (block_fwd(c, ts, ts.blocks[i], h->blocks[i], "layers_graph_conv." + std::to_string(i) + ".", s.Out, Fn)) return 1;
    cur = ts.blocks[i].Out;
    F = Fn; Tp = Tn;
  }
  ts.last = cur; ts.Flast = F;
  if (!c.dry && y) {
    const int Cl = C << L;
    const float* ws = c.L->get("shrink.weight", (int64_t)3 * Cl);
    if (!c.L->ok) return 1;
    shrink_kernel<<<cdiv(F * J * 32, 256), 256, 0, c.st>>>(cur, Cl, ws, y, F * J, Cl);
  }
  return 0;
}

// dy -> the parameter gradients (c.pgrad) and dL/dx into dx (B,T,J,F; may be null)
static int train_backward(gast_handle* h, TCtx& c, TrainState& ts, const float* dy, float* dx) {
  const gast_cfg& cf = h->cfg;
  const int J = c.J, C = cf.channels, L = cf.num_stages, Fin = cf.in_features, k0 = cf.filter_widths[0];
  const int Cl = C << L;
  long long F = ts.Flast;
  // shrink
  float* dcur = c.fl((size_t)F * J * Cl);
  if (!c.dry) {
    const float* ws = c.L->get("shrink.weight", (int64_t)3 * Cl);
    float* gws;
    if (!want_grad(c, "shrink.weight", (int64_t)3 * Cl, &gws) || !c.L->ok) return 1;
    shrink_bwd_x_kernel<<<cdiv(F * J * Cl, 256), 256, 0, c.st>>>(dy, ws, F * J, Cl, dcur);
    if (gws) shrink_bwd_w_kernel<<<cdiv(Cl, 32), dim3(32, SBW_RG), 0, c.st>>>(dy, ts.last, F * J, Cl, gws);
  }
  for (int i = L - 1; i >= 1; --i) {
    StageSave& s = ts.stages[i - 1];
    const int Cw = s.Cw;
    const long long Mn = s.Fout * J, Mi = s.Fin * J;
    float* dSout = c.fl((size_t)Mn * Cw);
    if (block_bwd(c, ts.blocks[i], h->blocks[i], dcur, dSout)) return 1;
    // stage: out = res + drop(relu(bn(conv1x1(h))));  h = relu(bn(conv_taps(x)))
    float* dXin = c.fl((size_t)Mi * Cw);
    float* dZ2 = c.fl((size_t)Mn * Cw);
    float* dHh = c.fl((size_t)Mn * Cw);
    float* dZ1 = c.fl((size_t)Mn * Cw);
    float* Xcol = c.fl((size_t)Mn * s.taps * Cw);
    float* dXcol = c.fl((size_t)Mn * s.taps * Cw);
    float* dWt = c.fl((size_t)Cw * s.taps * Cw);
    if (!c.dry) {
      cudaMemsetAsync(dXin, 0, sizeof(float) * (size_t)Mi * Cw, c.st);
      const ASeg rs = seg_taps(dXin, Cw, Cw, 1, 0, s.resmap);
      seg_scatter_add_kernel<<<cdiv(Mn * Cw, 256), 256, 0, c.st>>>(rs, J, s.Fout, dSout, Cw, 0);
    }
    if (bn_bwd(c, s.bnB, dSout, Cw, dZ2, Cw)) return 1;
    {
      const std::string k1s = "layers_conv." + std::to_string(2 * s.idx + 1) + ".weight";
      const float* w1 = c.dry ? nullptr : c.L->get(k1s, (int64_t)Cw * Cw);
      float* gw1;
      if (!want_grad(c, k1s, (int64_t)Cw * Cw, &gw1) || (!c.dry && !c.L->ok)) return 1;
      if (dense_tn(c, dZ2, Cw, s.Hh, Cw, Mn, Cw, Cw, gw1, Cw)) return 1;
      if (dense_nn(c, dZ2, Cw, w1, Cw, Mn, Cw, Cw, dHh, Cw)) return 1;
    }
    if (bn_bwd(c, s.bnA, dHh, Cw, dZ1, Cw)) return 1;
    const ASeg sg = seg_taps(s.X, Cw, Cw, s.taps, (long long)s.dil * J * Cw, s.tapmap);
    if (!c.dry && c.pgrad) seg_gather_kernel<<<cdiv(Mn * sg.K, 256), 256, 0, c.st>>>(sg, J, s.Fout, Xcol, s.taps * Cw, 0);
    if (dense_tn(c, dZ1, Cw, Xcol, s.taps * Cw, Mn, Cw, s.taps * Cw, dWt, s.taps * Cw)) return 1;
    if (dense_nn(c, dZ1, Cw, s.Wt, s.taps * Cw, Mn, Cw, s.taps * Cw, dXcol, s.taps * Cw)) return 1;
    float* gw0;
    if (!want_grad(c, "layers_conv." + std::to_string(2 * s.idx) + ".weight", (int64_t)Cw * Cw * s.taps, &gw0)) return 1;
    if (!c.dry) {
      if (gw0)
        conv_wgrad_relayout_kernel<<<cdiv((long long)Cw * Cw * s.taps, 256), 256, 0, c.st>>>(dWt, Cw, Cw, s.taps, s.taps * Cw, gw0);
      ASeg dsg = sg; dsg.base = dXin;
      seg_scatter_add_kernel<<<cdiv(Mn * dsg.K, 256), 256, 0, c.st>>>(dsg, J, s.Fout, dXcol, s.taps * Cw, 0);
    }
    dcur = dXin;
    F = s.Fin;
  }
  // first block
  const long long F0 = (long long)ts.B * ts.T0, M0 = F0 * J;
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
  float* gwe;
  if (!want_grad(c, "expand_conv.weight", (int64_t)C * Fin * k0, &gwe)) return 1;
  if (!c.dry) {
    if (gwe) conv_wgrad_relayout_kernel<<<cdiv((long long)C * Fin * k0, 256), 256, 0, c.st>>>(dWe8, C, Fin, k0, KP, gwe);
    cudaMemsetAsync(dxbn, 0, sizeof(float) * (size_t)Min * Fin, c.st);
    const ASeg sg = seg_taps(dxbn, Fin, Fin, k0, (long long)J * Fin, RowMap{ts.T0, ts.T, ts.s0, 0});
    seg_scatter_add_kernel<<<cdiv(M0 * sg.K, 256), 256, 0, c.st>>>(sg, J, F0, dAcol, KP, 0);
  }
  // init_bn: dx = dxbn . gamma . invstd (frozen), the batch-statistics adjoint otherwise
  if (bn_bwd(c, ts.bnin, dxbn, Fin, dx ? dx : dxin, Fin)) return 1;
  return 0;
}
