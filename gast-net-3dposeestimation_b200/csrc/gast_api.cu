// libgast_b200: C ABI (include/gast_b200.h) + launch planning of the GAST-Net lifting path.
//
// Layout: every activation is channels-last, rows = (clip, frame, joint), fp32.  The
// reference's (B,C,T,N) <-> (B,T,N,C) permutes (gast_net.py:24,31,162; local_attention.py:136,149;
// global_attention.py:109,114,121,128) therefore vanish.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <type_traits>
#include <unordered_map>
#include <vector>

#include "../../include/gast_b200.h"
#include "gast_common.cuh"
#include "gemm_ffma.cuh"
#include "kernels_misc.cuh"
#include "gemm_tc.cuh"
#include "kernels_hbm.cuh"
#include "train_kernels.cuh"
#include "wgrad_tc.cuh"
#include "train_state.cuh"

using namespace gast;

// ------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";

static int fail(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return 1;
}

#define CUDA_OK(expr)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess)                                                              \
      return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

extern "C" const char* gast_last_error(void) { return g_err; }
extern "C" const char* gast_version(void) {
  return "gast_b200 0.5 (sm_90a; wgmma 3xFP16 on power-of-two-scaled operands, training 3xTF32)";
}

// ------------------------------------------------------------------------------------------
// handle
// ------------------------------------------------------------------------------------------
struct Binding {
  void* ptr;
  int64_t numel;
};

struct BlockConsts {   // derived, eval mode; all device pointers owned by the handle
  int C = 0;           // input width
  int Cout = 0;        // SemCH out width (== C inside a block)
  int heads = 0, Cg = 0;
  int tpm = 0;         // 64-channel tiles per mask
  float *Wloc = nullptr, *coef[2] = {nullptr, nullptr}, *shift_loc = nullptr;
  float *Wlc = nullptr, *blc = nullptr;
  float *Wg = nullptr, *bg = nullptr, *U = nullptr, *cab = nullptr, *Ck = nullptr;
  float *Wgc = nullptr, *bgc = nullptr;
  float *Wbc = nullptr, *bbc = nullptr;
  TcWeights tc_loc, tc_lc, tc_g, tc_gc, tc_bc;   // hi/lo split copies for the tensor-core core
};

struct StageConsts {
  int Cw = 0, taps = 0, stride = 1, dil = 1;
  float *Wt = nullptr, *bt = nullptr, *W1 = nullptr, *b1 = nullptr;
  TcWeights tc_t, tc_1;
  std::vector<float*> Wrot;          // streaming (stream.cuh): tap-rotated copies of Wt, one per rotation
  std::vector<TcWeights> tc_rot;
};

template <typename Rec>
struct AuditHook {   // one test-only launch audit of a handle: its callback, running index and captured-launch count
  int (*fn)(int32_t phase, const Rec* d, void* user) = nullptr;
  void* user = nullptr;
  long long index = 0;
  long long skips = 0;
};

struct gast_handle {
  gast_cfg cfg;
  std::vector<int32_t> sym_r, sym_c, con_r, con_c;
  NbrTable nbr[2];
  int nnz[2] = {0, 0};
  std::unordered_map<std::string, Binding> bound;
  std::unordered_map<std::string, Binding> grads;   // gradient outputs by state_dict key (training)
  // saved-for-backward state of the training forwards still waiting for their backward, keyed by the
  // caller's workspace (which holds the saved activations): several forwards may be outstanding
  // (micro-batches summed before .backward(), a logging forward under no_grad in between)
  std::vector<std::pair<void*, TrainState>> trains;
  std::vector<void*> owned;          // cudaMalloc'ed derived buffers
  std::vector<BlockConsts> blocks;
  std::vector<StageConsts> stages;
  std::vector<int> pad, shift;       // gast_net.py:57,136-143
  float *We = nullptr, *be = nullptr;
  bool prepared = false;
  bool stream_ready = false;         // tap-rotated stage weights match the current parameters
  unsigned long long* dropout_state = nullptr;   // caller-owned device counter added to the dropout seed (graph replays)
  int launches = 0;
  int tc_launches = 0;
  int gemm_core = 0;                 // 0 auto (tensor cores where possible), 1 force FFMA
  int precision = 0;                 // 0 fp32-grade (3xFP16 on scaled operands in inference, 3xTF32 in training),
                                     // 1 single-pass TF32 (inference only), 16 fp16 (inference only: the half form's
                                     // arithmetic and fp16 activations behind float32 x and y, with_types)
  int act_dtype = GAST_F32;          // activation type of the model forward (gast_set_activation_dtype)
  int train_precision = 0;           // training and every gradient: 0 fp32-grade, 1 single-pass TF32 (forward and
                                     // input-gradient GEMMs) with the TF32 weight-gradient kernel (wgrad_tc.cuh)
  int wgrad_tc_launches = 0;         // weight gradients of the last training call that ran on wgrad_tc_kernel
  // training: per-GEMM tensor-core operand copies (3xTF32), indexed by the GEMM's position in the step (train.cuh)
  std::vector<TcWeights> train_tc;
  // optional per-launch device timing (bench.py roofline): event pairs around every launch
  bool timing = false;
  std::vector<cudaEvent_t> ev_pool;
  std::vector<int> ev_kind;          // kind per recorded launch
  size_t ev_used = 0;
  int fpt = 0;
  int sm_count = 132;
  // test-only launch audits (gast_debug_set_gemm_audit, gast_debug_set_kernel_audit): called around every launch_gemm,
  // and every expand, row-dot, attention-mix and shrink launch, outside graph capture
  AuditHook<gast_gemm_audit> gemm_audit;
  AuditHook<gast_kernel_audit> kernel_audit;
};

constexpr int GAST_MAX_PENDING_TRAIN = 16;   // training forwards that may wait for their backward per handle

enum { LK_EXPAND = 0, LK_GEMM_PLAIN = 1, LK_GEMM_SEMCH = 2, LK_GEMM_GLOBAL = 3, LK_ROWDOT = 4, LK_SHRINK = 5,
       LK_TC_PLAIN = 6, LK_TC_SEMCH = 7, LK_TC_GLOBAL = 8, LK_GLOBAL_MIX = 9 };

template <typename T>
struct Elem { using type = T; };   // an element type as a value, for with_types' callback

template <typename T>
constexpr int32_t elem_dtype = std::is_same<T, __half>::value ? GAST_F16 : GAST_F32;   // the audit records' type code

// The element types of an inference forward or stream call, and the only reading of act_dtype and precision that picks
// them: f(Elem<Io>(), Elem<Act>()) with Io the type of the model's x and y and Act that of the activations between
// layers.  A half model (act_dtype) has both fp16; the fp16 precision has fp16 activations behind float32 x and y (and
// the streams' input history); else both are float32.  Training and every gradient keep fp32 activations at any
// inference precision (they run only where precision_check lets them) and do not call this.
template <typename F>
static auto with_types(const gast_handle* h, F f) {
  if (h->act_dtype == GAST_F16) return f(Elem<__half>(), Elem<__half>());
  if (h->precision == 16) return f(Elem<float>(), Elem<__half>());
  return f(Elem<float>(), Elem<float>());
}

static size_t act_esize(const gast_handle* h) {
  return with_types(h, [](auto, auto act) { return sizeof(typename decltype(act)::type); });
}

// The refusal of every entry that half does not run: training, every backward, the streams, the mpjpe forward
static int half_check(const gast_handle* h, const char* who) {
  if (h->act_dtype == GAST_F16)
    return fail("%s: the handle's activation type is fp16 (gast_set_activation_dtype), which runs the eval-mode forward "
                "and the chunked forward only; set GAST_F32 to train, differentiate, stream or take the mpjpe", who);
  return 0;
}

struct TimedLaunch {   // RAII: event pair around one launch when timing is on
  gast_handle* h; cudaStream_t st; bool on;
  TimedLaunch(gast_handle* h_, cudaStream_t st_, int kind) : h(h_), st(st_), on(h_->timing) {
    if (!on) return;
    while (h->ev_pool.size() < h->ev_used + 2) {
      cudaEvent_t e; cudaEventCreate(&e); h->ev_pool.push_back(e);
    }
    h->ev_kind.push_back(kind);
    cudaEventRecord(h->ev_pool[h->ev_used], st);
  }
  ~TimedLaunch() {
    if (!on) return;
    cudaEventRecord(h->ev_pool[h->ev_used + 1], st);
    h->ev_used += 2;
  }
};

static int dalloc(gast_handle* h, float** p, size_t nfloats) {
  void* q = nullptr;
  CUDA_OK(cudaMalloc(&q, (nfloats ? nfloats : 1) * sizeof(float)));
  CUDA_OK(cudaMemset(q, 0, (nfloats ? nfloats : 1) * sizeof(float)));
  h->owned.push_back(q);
  *p = reinterpret_cast<float*>(q);
  return 0;
}

static int build_nbr(const std::vector<int32_t>& r, const std::vector<int32_t>& c, int J, NbrTable* t) {
  if (J > 32 || r.size() > 160) return fail("mask too large (J=%d nnz=%zu)", J, r.size());
  memset(t, 0, sizeof(*t));
  int z = 0;
  for (int i = 0; i < J; ++i) {
    t->row_ptr[i] = (unsigned char)z;
    while (z < (int)r.size() && r[z] == i) {
      if (z > 0 && r[z - 1] == i && c[z - 1] >= c[z]) return fail("mask nonzeros not in row-major order");
      t->col[z] = (unsigned char)c[z];
      ++z;
    }
    if (z == t->row_ptr[i]) return fail("mask row %d is empty (softmax over nothing)", i);
  }
  if (z != (int)r.size()) return fail("mask nonzeros not in row-major order");
  t->row_ptr[J] = (unsigned char)z;
  return 0;
}

static int alloc_block(gast_handle* h, BlockConsts* b, int C, int Cout, int heads, int Cg, int kind) {
  b->C = C; b->Cout = Cout; b->heads = heads; b->Cg = Cg;
  b->tpm = (Cout + 63) / 64;
  const bool has_local = (kind == GAST_KIND_MODEL || kind == GAST_KIND_BLOCK || kind == GAST_KIND_LOCAL ||
                          kind == GAST_KIND_SEMCH);
  const bool has_global = (kind == GAST_KIND_MODEL || kind == GAST_KIND_BLOCK || kind == GAST_KIND_MGLOBAL ||
                           kind == GAST_KIND_GLOBAL_HEAD);
  const int nmask = (kind == GAST_KIND_SEMCH) ? 1 : 2;
  if (has_local) {
    if (dalloc(h, &b->Wloc, (size_t)nmask * b->tpm * 128 * C)) return 1;
    for (int m = 0; m < nmask; ++m)
      if (dalloc(h, &b->coef[m], (size_t)h->nnz[m] * Cout)) return 1;
    if (dalloc(h, &b->shift_loc, (size_t)nmask * Cout)) return 1;
    if (kind != GAST_KIND_SEMCH) {
      if (dalloc(h, &b->Wlc, (size_t)C * 2 * C) || dalloc(h, &b->blc, C)) return 1;
    }
  }
  if (has_global) {
    const int Ng = heads * Cg;
    if (dalloc(h, &b->Wg, (size_t)Ng * C) || dalloc(h, &b->bg, Ng) || dalloc(h, &b->U, (size_t)2 * heads * C) ||
        dalloc(h, &b->cab, 2 * heads) || dalloc(h, &b->Ck, (size_t)heads * h->cfg.num_joints * h->cfg.num_joints))
      return 1;
    if (kind != GAST_KIND_GLOBAL_HEAD) {
      if (dalloc(h, &b->Wgc, (size_t)C * C) || dalloc(h, &b->bgc, C)) return 1;
    }
  }
  if (kind == GAST_KIND_MODEL || kind == GAST_KIND_BLOCK) {
    if (dalloc(h, &b->Wbc, (size_t)2 * C * 3 * C) || dalloc(h, &b->bbc, 2 * C)) return 1;
  }
  return 0;
}

extern "C" int gast_create(gast_t** out, const gast_cfg* cfg) {
  if (!out || !cfg) return fail("gast_create: null argument");
  *out = nullptr;
  const int J = cfg->num_joints;
  if (J < 2 || J > 32) return fail("gast_create: num_joints %d out of range", J);
  if (cfg->channels <= 0 || cfg->channels % 4) return fail("gast_create: channels must be a positive multiple of 4");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail("gast_create: no CUDA device (this library has no CPU path)");
  CUDA_OK(cudaSetDevice(cfg->device));
  cudaDeviceProp prop;
  CUDA_OK(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) return fail("gast_create: built for sm_90a, device is sm_%d%d", prop.major, prop.minor);

  gast_handle* h = new gast_handle();
  h->cfg = *cfg;
  h->sm_count = prop.multiProcessorCount;
  h->fpt = 128 / J;
  h->sym_r.assign(cfg->sym_rows, cfg->sym_rows + cfg->sym_nnz);
  h->sym_c.assign(cfg->sym_cols, cfg->sym_cols + cfg->sym_nnz);
  h->nnz[0] = cfg->sym_nnz;
  const int kind = cfg->kind;
  const bool need_sym = (kind != GAST_KIND_MGLOBAL && kind != GAST_KIND_GLOBAL_HEAD);
  const bool need_con = (kind == GAST_KIND_MODEL || kind == GAST_KIND_BLOCK || kind == GAST_KIND_LOCAL);
  if (need_con) {
    h->con_r.assign(cfg->con_rows, cfg->con_rows + cfg->con_nnz);
    h->con_c.assign(cfg->con_cols, cfg->con_cols + cfg->con_nnz);
    h->nnz[1] = cfg->con_nnz;
  }
  h->cfg.sym_rows = h->cfg.sym_cols = h->cfg.con_rows = h->cfg.con_cols = nullptr;
  int rc = 0;
  if (need_sym) rc |= build_nbr(h->sym_r, h->sym_c, J, &h->nbr[0]);
  if (need_con) rc |= build_nbr(h->con_r, h->con_c, J, &h->nbr[1]);
  if (rc) { delete h; return 1; }

  if (kind == GAST_KIND_MODEL) {
    const int L = cfg->num_stages;
    if (L < 1 || L > GAST_MAX_STAGES) { delete h; return fail("gast_create: num_stages %d", L); }
    for (int i = 0; i < L; ++i)
      if (cfg->filter_widths[i] % 2 == 0) { delete h; return fail("Only odd filter widths are supported"); }
    const int C = cfg->channels;
    // geometry, gast_net.py:57,136-143 / 213-220
    h->pad.push_back(cfg->filter_widths[0] / 2);
    h->shift.push_back(cfg->causal ? cfg->filter_widths[0] / 2 : 0);
    int nd = cfg->filter_widths[0];
    h->blocks.resize(L);
    h->stages.resize(L - 1);
    rc |= alloc_block(h, &h->blocks[0], C, C, 4, C / 4, kind);
    for (int i = 1; i < L; ++i) {
      const int fw = cfg->filter_widths[i];
      const int Cw = C << i;
      h->pad.push_back((fw - 1) * nd / 2);
      StageConsts& s = h->stages[i - 1];
      s.Cw = Cw;
      if (cfg->strided) {
        h->shift.push_back(cfg->causal ? fw / 2 : 0);
        s.taps = fw; s.stride = fw; s.dil = 1;
      } else {
        h->shift.push_back(cfg->causal ? (fw / 2) * nd : 0);
        if (cfg->dense) { s.taps = 2 * h->pad.back() + 1; s.stride = 1; s.dil = 1; }
        else { s.taps = fw; s.stride = 1; s.dil = nd; }
      }
      rc |= dalloc(h, &s.Wt, (size_t)Cw * s.taps * Cw) | dalloc(h, &s.bt, Cw) |
            dalloc(h, &s.W1, (size_t)Cw * Cw) | dalloc(h, &s.b1, Cw);
      rc |= alloc_block(h, &h->blocks[i], Cw, Cw, 4, Cw / 4, kind);
      nd *= fw;
    }
    rc |= dalloc(h, &h->We, (size_t)C * cfg->filter_widths[0] * cfg->in_features) | dalloc(h, &h->be, C);
  } else {
    h->blocks.resize(1);
    const int C = cfg->channels;
    int Cout = C, heads = 4, Cg = C / 4;
    if (kind == GAST_KIND_SEMCH) Cout = cfg->channels_out > 0 ? cfg->channels_out : C;
    if (kind == GAST_KIND_MGLOBAL) { heads = cfg->heads; Cg = C / heads; }
    if (kind == GAST_KIND_GLOBAL_HEAD) { heads = 1; Cg = cfg->channels_out; }
    if (heads < 1 || heads > 4) { delete h; return fail("gast_create: heads=%d unsupported (1..4)", heads); }
    if (Cout % 4 || (heads * Cg) % 4) { delete h; return fail("gast_create: widths must be multiples of 4"); }
    rc |= alloc_block(h, &h->blocks[0], C, Cout, heads, Cg, kind);
  }
  if (rc) { gast_destroy(h); return 1; }
  *out = h;
  return 0;
}

extern "C" void gast_destroy(gast_t* h) {
  if (!h) return;
  for (void* p : h->owned) cudaFree(p);
  for (cudaEvent_t e : h->ev_pool) cudaEventDestroy(e);
  delete h;
}

extern "C" int gast_bind(gast_t* h, int32_t n, const char* const* keys, void* const* ptrs, const int64_t* numel) {
  if (!h) return fail("gast_bind: null handle");
  for (int i = 0; i < n; ++i) h->bound[keys[i]] = Binding{ptrs[i], numel[i]};
  h->prepared = false;
  return 0;
}

extern "C" int gast_set_gemm_core(gast_t* h, int32_t core) {
  if (!h) return fail("null handle");
  if (core != 0 && core != 1) return fail("gast_set_gemm_core: core must be 0 (auto) or 1 (ffma)");
  if (core == 1 && h->act_dtype == GAST_F16)
    return fail("gast_set_gemm_core: the activation type is fp16 (gast_set_activation_dtype), which runs on the "
                "tensor-core core only");
  if (core == 1 && h->precision == 16)
    return fail("gast_set_gemm_core: the precision is fp16 (gast_set_precision(h, 16)), which runs on the tensor-core "
                "core only");
  h->gemm_core = core;
  return 0;
}

extern "C" int gast_set_precision(gast_t* h, int32_t mode) {
  if (!h) return fail("null handle");
  if (mode != 0 && mode != 1 && mode != 16)
    return fail("gast_set_precision: mode must be 0 (fp32-grade), 1 (tf32) or 16 (fp16), got %d", mode);
  if (mode == 1 && h->act_dtype == GAST_F16)
    return fail("gast_set_precision: the activation type is fp16 (gast_set_activation_dtype), which has its own "
                "arithmetic; TF32 needs GAST_F32");
  if (mode == 16) {   // the half form's arithmetic: its limits (gast_set_activation_dtype) apply
    if (h->act_dtype == GAST_F16)
      return fail("gast_set_precision: fp16 precision is for float32 models; the activation type is already fp16 "
                  "(gast_set_activation_dtype), which has its own fp16 arithmetic");
    if (h->cfg.kind != GAST_KIND_MODEL)
      return fail("gast_set_precision: fp16 precision runs the whole model (MODEL kind) only, not a sub-module");
    if (h->gemm_core != 0)
      return fail("gast_set_precision: fp16 precision runs on the tensor-core core only (gast_set_gemm_core(h, 0))");
    if (h->cfg.channels % TC_KS)
      return fail("gast_set_precision: fp16 precision needs channels that are a multiple of %d (got %d): there is no "
                  "FFMA core in fp16", TC_KS, h->cfg.channels);
    if (h->cfg.num_joints > MIX_JMAX)
      return fail("gast_set_precision: fp16 precision takes at most %d joints (got %d)", MIX_JMAX, h->cfg.num_joints);
  }
  h->precision = mode;
  return 0;
}

extern "C" int gast_set_activation_dtype(gast_t* h, int32_t dtype) {
  if (!h) return fail("null handle");
  if (dtype != GAST_F32 && dtype != GAST_F16)
    return fail("gast_set_activation_dtype: dtype must be GAST_F32 (0) or GAST_F16 (1), got %d", dtype);
  if (dtype == GAST_F16) {
    if (h->cfg.kind != GAST_KIND_MODEL)
      return fail("gast_set_activation_dtype: fp16 runs the whole model (MODEL kind) only, not a sub-module");
    if (h->precision != 0)
      return fail("gast_set_activation_dtype: fp16 needs gast_set_precision(h, 0), not TF32 or the fp16 precision "
                  "(precision is %d)", h->precision);
    if (h->cfg.num_joints > MIX_JMAX)   // the attention then needs the fused GLOBAL epilogue, not offered in half
      return fail("gast_set_activation_dtype: fp16 takes at most %d joints (got %d)", MIX_JMAX, h->cfg.num_joints);
    if (h->cfg.channels % TC_KS)   // every GEMM width is a multiple of channels; the half form takes multiples of 32
      return fail("gast_set_activation_dtype: fp16 needs channels that are a multiple of %d (got %d): there is no FFMA "
                  "core in half", TC_KS, h->cfg.channels);
    if (h->gemm_core != 0) return fail("gast_set_activation_dtype: fp16 runs on the tensor-core core only "
                                       "(gast_set_gemm_core(h, 0))");
  }
  h->act_dtype = dtype;
  return 0;
}

extern "C" int gast_set_train_precision(gast_t* h, int32_t mode) {
  if (!h) return fail("null handle");
  if (mode != 0 && mode != 1)
    return fail("gast_set_train_precision: mode must be 0 (fp32-grade) or 1 (tf32), got %d", mode);
  h->train_precision = mode;
  return 0;
}

extern "C" int32_t gast_last_launch_count(const gast_t* h) { return h ? h->launches : -1; }
extern "C" int32_t gast_last_wgrad_tc_launch_count(const gast_t* h) { return h ? h->wgrad_tc_launches : -1; }
extern "C" int32_t gast_last_tc_launch_count(const gast_t* h) { return h ? h->tc_launches : -1; }

extern "C" int gast_set_timing(gast_t* h, int32_t on) {
  if (!h) return fail("null handle");
  h->timing = on != 0;
  return 0;
}

extern "C" int32_t gast_get_timings(gast_t* h, int32_t max_n, float* ms, int32_t* kinds) {
  if (!h) return -1;
  int n = (int)(h->ev_used / 2);
  if (n > max_n) n = max_n;
  for (int i = 0; i < n; ++i) {
    if (cudaEventSynchronize(h->ev_pool[2 * i + 1]) != cudaSuccess) return -1;
    float t = 0.f;
    cudaEventElapsedTime(&t, h->ev_pool[2 * i], h->ev_pool[2 * i + 1]);
    ms[i] = t;
    kinds[i] = h->ev_kind[i];
  }
  return n;
}

// ------------------------------------------------------------------------------------------
// prepare
// ------------------------------------------------------------------------------------------
// Finds the parameters (or, with grads, the gradient buffers) bound on a handle by state_dict key.  The first failed
// lookup sets the error and is kept in `err`; ok stays false from then on.
struct Lookup {
  const std::unordered_map<std::string, Binding>& m;
  const char* what;
  bool ok = true;
  std::string err;
  // optional: every key asked for, once each, with the element count asked, in the order of its first lookup
  std::vector<std::pair<std::string, int64_t>>* asked = nullptr;
  explicit Lookup(gast_handle* h, bool grads = false)
      : m(grads ? h->grads : h->bound), what(grads ? "gradient buffer" : "parameter") {}
  Lookup(const std::unordered_map<std::string, Binding>& map, const char* what_) : m(map), what(what_) {}
  float* get(const std::string& key, int64_t numel) {
    if (asked && std::none_of(asked->begin(), asked->end(), [&](const auto& a) { return a.first == key; }))
      asked->emplace_back(key, numel);
    auto it = m.find(key);
    if (it != m.end() && (numel < 0 || it->second.numel == numel)) return reinterpret_cast<float*>(it->second.ptr);
    if (ok) {
      if (it == m.end()) fail("%s '%s' is not bound", what, key.c_str());
      else fail("%s '%s' has %lld elements, expected %lld", what, key.c_str(), (long long)it->second.numel, (long long)numel);
      err = g_err;
    }
    ok = false;
    return nullptr;
  }
  BnP bn(const std::string& prefix, int C) {
    BnP b;
    b.w = get(prefix + "weight", C); b.b = get(prefix + "bias", C);
    b.rm = get(prefix + "running_mean", C); b.rv = get(prefix + "running_var", C);
    return b;
  }
};

static inline unsigned cdiv(long long a, long long b) { return (unsigned)((a + b - 1) / b); }

static int prep_conv(cudaStream_t st, float* out, float* bias, const float* w, int N, int Cin, int taps, BnP bn) {
  long long total = (long long)N * Cin * taps;
  fold_conv_kernel<<<cdiv(total, 256), 256, 0, st>>>(out, bias, w, N, Cin, taps, bn);
  return 0;
}

static int prepare_local(gast_handle* h, Lookup& L, cudaStream_t st, BlockConsts& b, const std::string& lp, int kind) {
  const int C = b.C, Co = b.Cout, J = h->cfg.num_joints;
  const int nmask = (kind == GAST_KIND_SEMCH) ? 1 : 2;
  for (int m = 0; m < nmask; ++m) {
    std::string gp = (kind == GAST_KIND_SEMCH) ? lp : lp + (m == 0 ? "gcn_sym." : "gcn_con.");
    const float* W = L.get(gp + "W", (int64_t)2 * C * Co);
    const bool shared = (kind == GAST_KIND_SEMCH) && h->cfg.semch_shared_e;
    const float* e = L.get(gp + "e", shared ? h->nnz[m] : (int64_t)Co * h->nnz[m]);
    BnP bn = {nullptr, nullptr, nullptr, nullptr};
    const float* bias = nullptr;
    if (kind != GAST_KIND_SEMCH) bn = L.bn(lp + (m == 0 ? "bn_1." : "bn_2."), Co);
    else if (h->cfg.semch_bias) bias = L.get(gp + "bias", Co);
    if (!L.ok) return 1;
    long long tot = (long long)b.tpm * 128 * C;
    semch_pack_kernel<<<cdiv(tot, 256), 256, 0, st>>>(b.Wloc + (size_t)m * b.tpm * 128 * C, W, b.tpm, C, Co);
    semch_coef_kernel<<<cdiv((long long)Co * J, 128), 128, 0, st>>>(
        b.coef[m], b.shift_loc + (size_t)m * Co, e, shared ? 0 : h->nnz[m], h->nbr[m], h->nnz[m], Co, J, bn, bias);
  }
  if (kind != GAST_KIND_SEMCH) {
    const float* w = L.get(lp + "cat_conv.weight", (int64_t)C * 2 * C);
    BnP bn = L.bn(lp + "cat_bn.", C);
    if (!L.ok) return 1;
    prep_conv(st, b.Wlc, b.blc, w, C, 2 * C, 1, bn);
  }
  return 0;
}

struct GlobalParams {   // what prepare_global reads: each head's parameters, then the cat conv and its BatchNorm
  const float *gw[4], *gb[4], *tw[4], *tb[4], *pw[4], *pb[4], *wc[4], *ck[4];
  const float* cat_w = nullptr;
  BnP cat_bn = {nullptr, nullptr, nullptr, nullptr};
};

static void global_params(const gast_handle* h, Lookup& L, const BlockConsts& b, const std::string& gp, int kind,
                          GlobalParams* p) {
  const int C = b.C, J = h->cfg.num_joints, Cg = b.Cg;
  for (int hd = 0; hd < b.heads; ++hd) {
    std::string hp = (kind == GAST_KIND_GLOBAL_HEAD) ? gp : gp + "attentions." + std::to_string(hd) + ".";
    // theta / phi are inter_channels wide; in a block inter == Cg (global_attention.py:21-24)
    p->gw[hd] = L.get(hp + "g.weight", (int64_t)Cg * C);
    p->gb[hd] = L.get(hp + "g.bias", Cg);
    p->tw[hd] = L.get(hp + "theta.weight", (int64_t)Cg * C);
    p->tb[hd] = L.get(hp + "theta.bias", Cg);
    p->pw[hd] = L.get(hp + "phi.weight", (int64_t)Cg * C);
    p->pb[hd] = L.get(hp + "phi.bias", Cg);
    p->wc[hd] = L.get(hp + "concat_project.0.weight", 2 * Cg);
    p->ck[hd] = L.get(hp + "C_k", (int64_t)J * J);
  }
  if (kind != GAST_KIND_GLOBAL_HEAD) {
    p->cat_w = L.get(gp + "cat_conv.weight", (int64_t)C * C);
    p->cat_bn = L.bn(gp + "cat_bn.", C);
  }
}

// the eval constants of a global layer from the parameters global_params found
static int prepare_global(const gast_handle* h, cudaStream_t st, BlockConsts& b, const GlobalParams& p, int kind) {
  const int C = b.C, J = h->cfg.num_joints, Cg = b.Cg;
  for (int hd = 0; hd < b.heads; ++hd) {
    CUDA_OK(cudaMemcpyAsync(b.Wg + (size_t)hd * Cg * C, p.gw[hd], sizeof(float) * Cg * C, cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(b.bg + (size_t)hd * Cg, p.gb[hd], sizeof(float) * Cg, cudaMemcpyDeviceToDevice, st));
    CUDA_OK(cudaMemcpyAsync(b.Ck + (size_t)hd * J * J, p.ck[hd], sizeof(float) * J * J, cudaMemcpyDeviceToDevice, st));
    global_collapse_kernel<<<cdiv(C, 32), 256, 0, st>>>(b.U, b.cab, p.tw[hd], p.tb[hd], p.pw[hd], p.pb[hd], p.wc[hd], hd,
                                                        C, Cg);
  }
  if (kind != GAST_KIND_GLOBAL_HEAD) prep_conv(st, b.Wgc, b.bgc, p.cat_w, C, C, 1, p.cat_bn);
  return 0;
}

static int prepare_block(gast_handle* h, Lookup& L, cudaStream_t st, BlockConsts& b, const std::string& P) {
  if (prepare_local(h, L, st, b, P + "local_graph_layer.", GAST_KIND_BLOCK)) return 1;
  GlobalParams gpar;
  global_params(h, L, b, P + "global_graph_layer.", GAST_KIND_BLOCK, &gpar);
  if (!L.ok || prepare_global(h, st, b, gpar, GAST_KIND_BLOCK)) return 1;
  const int C = b.C;
  const float* w = L.get(P + "cat_conv.weight", (int64_t)2 * C * 3 * C);
  BnP bn = L.bn(P + "cat_bn.", 2 * C);
  if (!L.ok) return 1;
  prep_conv(st, b.Wbc, b.bbc, w, 2 * C, 3 * C, 1, bn);
  return 0;
}

// ------------------------------------------------------------------------------------------
// tensor-core weight copies
// ------------------------------------------------------------------------------------------
static int prep_one_tc(gast_handle* h, cudaStream_t st, TcWeights& t, const float* W, int N, int K) {
  if (!W) return 0;
  int rc = tc_prepare_weights(t, W, N, K, st, &h->owned, true);   // inference: F16X3 at fp32 grade
  if (rc) return fail("tensor-core weight preparation failed: %s", cudaGetErrorString((cudaError_t)rc));
  return 0;
}

static int prepare_tc(gast_handle* h, cudaStream_t st) {
  const int kind = h->cfg.kind;
  for (BlockConsts& b : h->blocks) {
    const int C = b.C;
    const int nmask = (kind == GAST_KIND_SEMCH) ? 1 : 2;
    if (prep_one_tc(h, st, b.tc_loc, b.Wloc, nmask * b.tpm * 128, C)) return 1;
    if (prep_one_tc(h, st, b.tc_lc, b.Wlc, C, 2 * C)) return 1;
    if (prep_one_tc(h, st, b.tc_g, b.Wg, b.heads * b.Cg, C)) return 1;
    if (prep_one_tc(h, st, b.tc_gc, b.Wgc, C, C)) return 1;
    if (prep_one_tc(h, st, b.tc_bc, b.Wbc, 2 * C, 3 * C)) return 1;
  }
  for (StageConsts& s : h->stages) {
    if (prep_one_tc(h, st, s.tc_t, s.Wt, s.Cw, s.taps * s.Cw)) return 1;
    if (prep_one_tc(h, st, s.tc_1, s.W1, s.Cw, s.Cw)) return 1;
  }
  return 0;
}

extern "C" int gast_prepare(gast_t* h, void* stream) {
  if (!h) return fail("gast_prepare: null handle");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUDA_OK(cudaSetDevice(h->cfg.device));
  Lookup L{h};
  const int kind = h->cfg.kind;
  if (kind == GAST_KIND_MODEL) {
    const int C = h->cfg.channels, Fin = h->cfg.in_features, k0 = h->cfg.filter_widths[0];
    const float* we = L.get("expand_conv.weight", (int64_t)C * Fin * k0);
    BnP bin = L.bn("init_bn.", Fin), bex = L.bn("expand_bn.", C);
    if (!L.ok) return 1;
    expand_fold_kernel<<<cdiv(C, 128), 128, 0, st>>>(h->We, h->be, we, C, Fin, k0, bin, bex);
    for (size_t i = 0; i < h->blocks.size(); ++i)
      if (prepare_block(h, L, st, h->blocks[i], "layers_graph_conv." + std::to_string(i) + ".")) return 1;
    for (size_t i = 0; i < h->stages.size(); ++i) {
      StageConsts& s = h->stages[i];
      const float* w0 = L.get("layers_conv." + std::to_string(2 * i) + ".weight", (int64_t)s.Cw * s.Cw * s.taps);
      const float* w1 = L.get("layers_conv." + std::to_string(2 * i + 1) + ".weight", (int64_t)s.Cw * s.Cw);
      BnP b0 = L.bn("layers_bn." + std::to_string(2 * i) + ".", s.Cw);
      BnP b1 = L.bn("layers_bn." + std::to_string(2 * i + 1) + ".", s.Cw);
      if (!L.ok) return 1;
      prep_conv(st, s.Wt, s.bt, w0, s.Cw, s.Cw, s.taps, b0);
      prep_conv(st, s.W1, s.b1, w1, s.Cw, s.Cw, 1, b1);
    }
    L.get("shrink.weight", (int64_t)3 * (C << (h->cfg.num_stages)));
    if (!L.ok) return 1;
  } else if (kind == GAST_KIND_BLOCK) {
    if (prepare_block(h, L, st, h->blocks[0], "")) return 1;
  } else if (kind == GAST_KIND_LOCAL || kind == GAST_KIND_SEMCH) {
    if (prepare_local(h, L, st, h->blocks[0], "", kind)) return 1;
  } else if (kind == GAST_KIND_MGLOBAL || kind == GAST_KIND_GLOBAL_HEAD) {
    GlobalParams gpar;
    global_params(h, L, h->blocks[0], "", kind, &gpar);
    if (!L.ok || prepare_global(h, st, h->blocks[0], gpar, kind)) return 1;
  } else {
    return fail("gast_prepare: unknown kind %d", kind);
  }
  if (prepare_tc(h, st)) return 1;
  CUDA_OK(cudaGetLastError());
  h->prepared = true;
  h->stream_ready = false;
  return 0;
}

// ------------------------------------------------------------------------------------------
// forward planning
// ------------------------------------------------------------------------------------------
// The schedule of a forward on clips of T frames.  It is the handle's own (cfg.strided) or, for a dilated model on a
// receptive-field-long clip, the equivalent strided one (same arithmetic per output, see SURVEY.md §7 "dense vs
// needed-only work").
static int geometry(const gast_handle* h, int T, int strided_now, Geometry* g) {
  const gast_cfg& c = h->cfg;
  if (strided_now && !c.strided && c.dense) return fail("dense model has no strided schedule");
  if (!strided_now && c.strided) return fail("Optimized1f handle only runs the strided schedule");
  const int k0 = c.filter_widths[0];
  g->s0 = strided_now ? k0 : 1;
  if (T < k0) return fail("input has %d frames, fewer than the first filter width %d", T, k0);
  g->T0 = (T - k0) / g->s0 + 1;
  int Tp = g->T0;
  g->stages.clear();
  for (int i = 1; i < c.num_stages; ++i) {
    const int fw = c.filter_widths[i];
    StageGeo s;
    int res_mul, res_off;
    if (strided_now) {
      // gast_net.py:222-224,243 ; causal shift of the strided form is fw//2 (:220)
      s.taps = fw; s.stride = fw; s.dil = 1;
      res_mul = fw;
      res_off = (c.causal ? fw / 2 : 0) + fw / 2;
    } else {
      const StageConsts& sc = h->stages[i - 1];
      s.taps = sc.taps; s.stride = 1; s.dil = sc.dil;
      res_mul = 1;
      res_off = h->pad[i] + h->shift[i];   // gast_net.py:170
    }
    const int span = (s.taps - 1) * s.dil + 1;
    if (Tp < span) return fail("input of %d frames is shorter than the receptive field", T);
    const int Tn = (Tp - span) / s.stride + 1;
    // residual slice must cover the conv output (the reference would raise on the add otherwise)
    if (res_off + (long long)(Tn - 1) * res_mul >= Tp) return fail("residual slice out of range for T=%d", T);
    s.Tin = Tp; s.Tout = Tn;
    s.tapmap = RowMap{Tn, Tp, s.stride, 0};
    s.resmap = RowMap{Tn, Tp, res_mul, res_off};
    g->stages.push_back(s);
    Tp = Tn;
  }
  g->T_out = Tp;
  return 0;
}

extern "C" int32_t gast_receptive_field(const gast_t* h) {
  if (!h || h->cfg.kind != GAST_KIND_MODEL) return -1;
  int rf = 1;
  for (int p : h->pad) rf += 2 * p;
  return rf;
}

extern "C" int32_t gast_out_frames(const gast_t* h, int32_t T, int32_t strided_now) {
  if (!h) return -1;
  if (h->cfg.kind != GAST_KIND_MODEL) return T;
  Geometry g;
  if (geometry(h, T, strided_now, &g)) return -1;
  return g.T_out;
}

// workspace carve-up ------------------------------------------------------------------
struct Arena {
  char* base; size_t size; size_t off = 0; bool dry;
  size_t esize = sizeof(float);   // bytes per element of take(): 2 for the activations of a half forward (plan_model)
  float* take(size_t n) { return take_bytes(n * esize); }
  float* take32(size_t nfloats) { return take_bytes(nfloats * sizeof(float)); }
  float* take_bytes(size_t b) {
    size_t bytes = (b + 255) & ~(size_t)255;
    float* p = dry ? nullptr : reinterpret_cast<float*>(base + off);
    off += bytes;
    return p;
  }
};

// Caller buffers are used from their first 256-byte boundary; every *_bytes function adds at least that much slack.
static char* align256(void* p) {
  return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + 255) & ~(uintptr_t)255);
}

static Arena workspace_arena(void* workspace, size_t bytes, size_t off = 0) {
  return Arena{align256(workspace), bytes, off, false};
}

struct BlockBufs { float *XY, *L, *AB, *Y, *Gl; };

static void block_bufs(Arena& a, long long rows, int C, int Cout, int heads, int Cg, BlockBufs* b) {
  b->XY = a.take((size_t)rows * 2 * Cout);
  b->L = a.take((size_t)rows * C);
  b->AB = a.take((size_t)rows * 2 * heads);
  b->Y = a.take((size_t)rows * heads * Cg);
  b->Gl = a.take((size_t)rows * C);
}

// ------------------------------------------------------------------------------------------
// launches
// ------------------------------------------------------------------------------------------
// A operand of `taps` K-segments of width Kc, tap_stride floats apart; output row r reads input row map(r)
static ASeg seg_taps(const float* base, int ld, int Kc, int taps, long long tap_stride, RowMap map) {
  ASeg s; s.base = base; s.ld = ld; s.K = taps * Kc; s.Kc = Kc; s.tap_stride = tap_stride; s.map = map;
  return s;
}

static ASeg seg_flat(const float* base, int ld, int K) { return seg_taps(base, ld, K, 1, 0, RowMap{1, 1, 1, 0}); }

// GEMM over M plain rows: "frames" of one joint, 128 per tile, no residual
static void gemm_flat(GemmP& p, long long M) {
  memset(&p, 0, sizeof(p));
  p.F = (int)M; p.J = 1; p.fpt = 128;
  p.res_map = RowMap{1, 1, 1, 0};
}

static void gemm_defaults(GemmP& p, const gast_handle* h, long long F) {
  gemm_flat(p, F);
  p.J = h->cfg.num_joints; p.fpt = h->fpt;
}

// A 1x1 layer with flat operands and no joint mixing does not need frame-aligned tiles: run it as
// F*J "frames" of one joint, so that every tile carries 128 rows instead of floor(128/J)*J (119 for J=17).
static void gemm_defaults_flat(GemmP& p, const gast_handle* h, long long F) { gemm_flat(p, F * h->cfg.num_joints); }

static void audit_describe(const gast_gemm_audit& d, char* s, size_t n) {
  snprintf(s, n, "GEMM audit rejected launch %lld (epi %d, core %d, form %d, F %d J %d N %d K %d)", (long long)d.index,
           d.epi, d.core, d.tc_form, d.F, d.J, d.N, d.ldw);
}

static void audit_describe(const gast_kernel_audit& d, char* s, size_t n) {
  static const char* const kinds[] = {"expand", "rowdot", "mix", "shrink", "shrink_mpjpe"};
  snprintf(s, n, "kernel audit rejected launch %lld (%s, variant %d, rows %lld K %d)", (long long)d.index,
           kinds[d.kind], d.variant, (long long)d.rows, d.K);
}

// The host side of both test-only audits: launch() as it is when the hook is off, and, counted as a skip, under CUDA-graph
// capture (a callback cannot read a captured launch's operands); otherwise fill(d) writes the record and the hook's
// callback sees it just before and just after the launch, the stream synchronised each time.
template <typename Rec, typename Fill, typename Launch>
static int audited_launch(cudaStream_t st, AuditHook<Rec>& a, Fill fill, Launch launch) {
  if (!a.fn) return launch();
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  CUDA_OK(cudaStreamIsCapturing(st, &cs));
  if (cs != cudaStreamCaptureStatusNone) {
    a.skips++;
    return launch();
  }
  Rec d;
  memset(&d, 0, sizeof(d));
  fill(d);
  d.index = a.index++;
  for (int phase = 0; phase < 2; ++phase) {
    if (phase && launch()) return 1;
    CUDA_OK(cudaStreamSynchronize(st));
    if (a.fn(phase, &d, a.user)) {
      char s[256];
      audit_describe(d, s, sizeof(s));
      return fail("%s %s", s, phase ? "after it ran" : "before it ran");
    }
  }
  return 0;
}

// One expand, row-dot, attention-mix or shrink launch: audited, timed as `kind` (LK_*) and counted unless launch() refuses
template <typename Fill, typename Launch>
static int kernel_audited(gast_handle* h, cudaStream_t st, int kind, Fill fill, Launch launch) {
  return audited_launch(st, h->kernel_audit, [&](gast_kernel_audit& d) {
    d.gemm_index = h->gemm_audit.index;
    fill(d);
  }, [&] {
    TimedLaunch tl(h, st, kind);
    if (launch()) return 1;
    h->launches++;
    return 0;
  });
}

// the audit record of a launch (gast_gemm_audit mirrors GemmP); prec < 0: the FFMA core
static void gemm_audit_record(int epi, const GemmP& p, int prec, gast_gemm_audit* d) {
  d->epi = epi;
  d->core = prec < 0 ? 1 : 0;
  d->tc_form = prec;
  d->nseg = p.nseg;
  for (int s = 0; s < p.nseg; ++s) {
    const ASeg& a = p.seg[s];
    d->seg[s] = gast_gemm_audit_seg{a.base, a.tap_stride, a.ld, a.K, a.Kc, a.map.T_out, a.map.T_in, a.map.t_mul, a.map.t_off};
    if (prec >= 0 && (prec == TC_F16 ? tc_seg_tma_h(a) : tc_seg_tma(a))) d->tma_mask |= 1 << s;
  }
  d->W = p.W; d->ldw = p.ldw; d->N = p.N; d->F = p.F; d->J = p.J; d->fpt = p.fpt; d->ld_out = p.ld_out;
  d->out = p.out; d->bias = p.bias; d->relu = p.relu; d->res = p.res; d->res_ld = p.res_ld;
  d->res_T_out = p.res_map.T_out; d->res_T_in = p.res_map.T_in; d->res_t_mul = p.res_map.t_mul; d->res_t_off = p.res_map.t_off;
  d->coef[0] = p.coef[0]; d->coef[1] = p.coef[1]; d->shift = p.shift; d->C = p.C; d->tiles_per_mask = p.tiles_per_mask;
  for (int m = 0; m < 2; ++m) {
    memcpy(d->nbr_row_ptr[m], p.nbr[m].row_ptr, sizeof(d->nbr_row_ptr[m]));
    memcpy(d->nbr_col[m], p.nbr[m].col, sizeof(d->nbr_col[m]));
  }
  d->ab = p.ab; d->ck = p.ck; d->bg = p.bg; d->heads = p.heads; d->Cg = p.Cg;
}

static int launch_gemm_core(gast_handle* h, cudaStream_t st, int epi, const GemmP& p, const TcWeights* tcw, int prec) {
  if (prec >= 0) {
    TimedLaunch tl(h, st, LK_TC_PLAIN + epi);
    int rc = tc_launch(st, epi, p, *tcw, prec);
    if (rc) return fail("tensor-core gemm launch failed: %s", cudaGetErrorString((cudaError_t)rc));
    h->launches++;
    h->tc_launches++;
    return 0;
  }
  TimedLaunch tl(h, st, LK_GEMM_PLAIN + epi);
  dim3 grid(cdiv(p.F, p.fpt), cdiv(p.N, FF_BN));
  int hpt = 1;
  if (epi == EPI_GLOBAL) hpt = p.heads < 4 ? p.heads : 4;
  size_t smem = ffma_smem_bytes(epi, p.J, p.fpt, hpt);
  const auto kernel = with_epi(epi, [](auto e) { return gemm_ffma_kernel<decltype(e)::value>; });
  static bool attr_set_dev[64][3];          // the opt-in is per device (one handle per device in one process)
  bool& attr_done = attr_set_dev[h->cfg.device & 63][epi];
  if (!attr_done) {
    CUDA_OK(cudaFuncSetAttribute((const void*)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
    attr_done = true;
  }
  kernel<<<grid, FF_THREADS, smem, st>>>(p);
  h->launches++;
  return 0;
}

static int launch_gemm(gast_handle* h, cudaStream_t st, int epi, const GemmP& p, const TcWeights* tcw) {
  if (p.F <= 0) return 0;
  int Ktot = 0;
  for (int s = 0; s < p.nseg; ++s) Ktot += p.seg[s].K;
  if (Ktot != p.ldw) return fail("internal: K mismatch %d vs %d", Ktot, p.ldw);
  if (p.N % 4 || p.ld_out % 4) return fail("internal: N/ld_out must be multiples of 4");
  // training's operand copies (train_tcw, the only ones without the fp16 pair) run at the training precision
  int prec = (h->gemm_core == 0 && tcw && tc_supported(p, epi, *tcw))
                 ? tc_prec(*tcw, tcw->f16 ? h->precision : h->train_precision) : -1;
  // fp16 operands: the half form or nothing (there is no FFMA core in half).  Training's operand copies (null, or
  // without the fp16 pair) read fp32 activations at every inference precision.
  if (h->act_dtype == GAST_F16 || (h->precision == 16 && tcw && tcw->f16)) {
    if (!tcw || !tc_supported_h(p, epi, *tcw))
      return fail("fp16 forward: a GEMM (N %d, K %d, epilogue %d) is not taken by the tensor-core core (widths must be "
                  "multiples of 32)", p.N, p.ldw, epi);
    prec = TC_F16;
  }
  return audited_launch(st, h->gemm_audit, [&](gast_gemm_audit& d) { gemm_audit_record(epi, p, prec, &d); },
                        [&] { return launch_gemm_core(h, st, epi, p, tcw, prec); });
}

extern "C" int gast_debug_set_gemm_audit(gast_t* h, gast_gemm_audit_fn fn, void* user) {
  if (!h) return fail("gast_debug_set_gemm_audit: null handle");
  h->gemm_audit.fn = fn;
  h->gemm_audit.user = user;
  return 0;
}

extern "C" int64_t gast_debug_gemm_audit_skips(const gast_t* h) { return h ? h->gemm_audit.skips : -1; }

extern "C" int gast_debug_set_kernel_audit(gast_t* h, gast_kernel_audit_fn fn, void* user) {
  if (!h) return fail("gast_debug_set_kernel_audit: null handle");
  h->kernel_audit.fn = fn;
  h->kernel_audit.user = user;
  return 0;
}

extern "C" int64_t gast_debug_kernel_audit_skips(const gast_t* h) { return h ? h->kernel_audit.skips : -1; }

enum { KA_EXPAND = 0, KA_ROWDOT = 1, KA_MIX = 2, KA_SHRINK = 3, KA_SHRINK_MPJPE = 4 };

// Act: the element type of X (with_types' Act; training passes float).  The row dots stay fp32 (they feed the softmax).
template <typename Act>
static int launch_rowdot(gast_handle* h, cudaStream_t st, Elem<Act>, const float* X, int ldx, const BlockConsts& b,
                         float* ab, long long rows) {
  if (rows <= 0) return 0;
  constexpr bool f16 = std::is_same<Act, __half>::value;
  const int Q = 2 * b.heads;
  unsigned blocks = cdiv(rows * 32, 256);
  // rowdot8_kernel stages U in 48 KB of shared memory; its float32 form also reads X in float4 of 4 channels
  const bool r8 = Q == 8 && (size_t)8 * b.C * sizeof(float) <= 48 * 1024 && (f16 || b.C % 4 == 0);
  auto fill = [&](gast_kernel_audit& d) {
    d.kind = KA_ROWDOT; d.variant = r8 ? 0 : Q; d.block = (int)(&b - h->blocks.data());
    d.in_type = elem_dtype<Act>; d.x = X; d.U = b.U; d.cab = b.cab; d.ab = ab; d.rows = rows; d.K = b.C; d.ld = ldx;
    d.heads = b.heads;
  };
  return kernel_audited(h, st, LK_ROWDOT, fill, [&] {
    const Act* x = reinterpret_cast<const Act*>(X);
    if (r8) {
      unsigned g = (unsigned)std::min<long long>((rows * 32 + 255) / 256, (long long)h->sm_count * 8);
      rowdot8_kernel<<<g, 256, sizeof(float) * 8 * b.C, st>>>(x, ldx, b.U, b.cab, ab, rows, b.C);
    } else if (Q == 8) rowdot_kernel<8><<<blocks, 256, 0, st>>>(x, ldx, b.U, b.cab, ab, rows, b.C);
    else if constexpr (f16) return fail("internal: fp16 forward with heads=%d", b.heads);   // no fp16 form below
    else if (Q == 6) rowdot_kernel<6><<<blocks, 256, 0, st>>>(x, ldx, b.U, b.cab, ab, rows, b.C);
    else if (Q == 4) rowdot_kernel<4><<<blocks, 256, 0, st>>>(x, ldx, b.U, b.cab, ab, rows, b.C);
    else if (Q == 2) rowdot_kernel<2><<<blocks, 256, 0, st>>>(x, ldx, b.U, b.cab, ab, rows, b.C);
    else return fail("internal: heads=%d", b.heads);
    return 0;
  });
}

// SemCH (both masks) -> XY ; then local cat conv -> L          (local_attention.py:130-151)
static int run_local(gast_handle* h, cudaStream_t st, BlockConsts& b, const float* X, long long F,
                     const BlockBufs& w, float* out_L, int kind) {
  const int C = b.C, Co = b.Cout;
  const int nmask = (kind == GAST_KIND_SEMCH) ? 1 : 2;
  GemmP p;
  gemm_defaults(p, h, F);
  p.nseg = 1; p.seg[0] = seg_flat(X, C, C);
  p.W = b.Wloc; p.ldw = C; p.N = nmask * b.tpm * 128;
  p.out = (kind == GAST_KIND_SEMCH) ? out_L : w.XY;
  p.ld_out = nmask * Co;
  p.relu = (kind == GAST_KIND_SEMCH) ? 0 : 1;
  p.coef[0] = b.coef[0]; p.coef[1] = b.coef[1];
  p.shift = b.shift_loc; p.C = Co; p.tiles_per_mask = b.tpm;
  p.nbr[0] = h->nbr[0]; p.nbr[1] = h->nbr[1];
  if (launch_gemm(h, st, EPI_SEMCH, p, &b.tc_loc)) return 1;
  if (kind == GAST_KIND_SEMCH) return 0;
  gemm_defaults_flat(p, h, F);
  p.nseg = 1; p.seg[0] = seg_flat(w.XY, 2 * C, 2 * C);
  p.W = b.Wlc; p.ldw = 2 * C; p.N = C; p.out = out_L; p.ld_out = C; p.bias = b.blc; p.relu = 1;
  return launch_gemm(h, st, EPI_PLAIN, p, &b.tc_lc);
}

// collapsed theta/phi -> attention-mixed g -> Y ; then global cat conv -> Gl   (global_attention.py:52-130)
static int run_global(gast_handle* h, cudaStream_t st, BlockConsts& b, const float* X, long long F,
                      const BlockBufs& w, float* out_G, int kind) {
  const int C = b.C, J = h->cfg.num_joints, Ng = b.heads * b.Cg;
  if (with_types(h, [&](auto, auto act) { return launch_rowdot(h, st, act, X, C, b, w.AB, F * J); })) return 1;
  GemmP p;
  // tensor-core core, block / MultiGlobalGraph: plain `g` GEMM (flat 128-row tiles) into out_G as scratch, then the
  // attention mix as its own full-occupancy kernel into Y.  Measured faster than the mix fused into the GEMM
  // epilogue, which stays for the FFMA core, the single-head kind and the shapes the mix kernel does not take.
  if (h->gemm_core == 0 && kind != GAST_KIND_GLOBAL_HEAD && b.tc_g.ready && Ng % 4 == 0 && b.Cg % 4 == 0 &&
      J <= MIX_JMAX) {
    gemm_defaults_flat(p, h, F);
    p.nseg = 1; p.seg[0] = seg_flat(X, C, C);
    p.W = b.Wg; p.ldw = C; p.N = Ng; p.out = out_G; p.ld_out = Ng; p.bias = b.bg; p.relu = 0;
    if (launch_gemm(h, st, EPI_PLAIN, p, &b.tc_g)) return 1;
    const int GV = Ng / 4;   // threads per frame
    int fpb = GV >= MIX_THREADS ? 1 : MIX_THREADS / GV;
    fpb = std::max(1, std::min(fpb, (int)(40 * 1024 / (sizeof(float) * b.heads * J * MIX_JP))));   // attention rows fit 40 KB
    const size_t smem = sizeof(float) * (size_t)fpb * b.heads * J * MIX_JP;
    if (with_types(h, [&](auto, auto act) {
          using Act = typename decltype(act)::type;
          auto fill = [&](gast_kernel_audit& d) {
            d.kind = KA_MIX; d.fpb = fpb; d.block = (int)(&b - h->blocks.data());
            d.in_type = d.out_type = elem_dtype<Act>; d.x = out_G; d.ab = w.AB; d.Ck = b.Ck; d.out = w.Y;
            d.rows = F; d.K = Ng; d.ld = Ng; d.J = J; d.heads = b.heads; d.Cg = b.Cg;
          };
          return kernel_audited(h, st, LK_GLOBAL_MIX, fill, [&] {
            global_mix_kernel<<<cdiv(F, fpb), MIX_THREADS, smem, st>>>(reinterpret_cast<const Act*>(out_G), Ng, w.AB,
                                                                       b.Ck, reinterpret_cast<Act*>(w.Y), Ng, F, J,
                                                                       b.heads, b.Cg, fpb);
            return 0;
          });
        }))
      return 1;
    CUDA_OK(cudaGetLastError());
    gemm_defaults_flat(p, h, F);
    p.nseg = 1; p.seg[0] = seg_flat(w.Y, C, C);
    p.W = b.Wgc; p.ldw = C; p.N = C; p.out = out_G; p.ld_out = C; p.bias = b.bgc; p.relu = 1;
    return launch_gemm(h, st, EPI_PLAIN, p, &b.tc_gc);
  }
  gemm_defaults(p, h, F);
  p.nseg = 1; p.seg[0] = seg_flat(X, C, C);
  p.W = b.Wg; p.ldw = C; p.N = Ng;
  p.out = (kind == GAST_KIND_GLOBAL_HEAD) ? out_G : w.Y;
  p.ld_out = Ng;
  p.ab = w.AB; p.ck = b.Ck; p.bg = b.bg; p.heads = b.heads; p.Cg = b.Cg;
  if (launch_gemm(h, st, EPI_GLOBAL, p, &b.tc_g)) return 1;
  if (kind == GAST_KIND_GLOBAL_HEAD) return 0;
  gemm_defaults_flat(p, h, F);
  p.nseg = 1; p.seg[0] = seg_flat(w.Y, C, C);
  p.W = b.Wgc; p.ldw = C; p.N = C; p.out = out_G; p.ld_out = C; p.bias = b.bgc; p.relu = 1;
  return launch_gemm(h, st, EPI_PLAIN, p, &b.tc_gc);
}

// GraphAttentionBlock (gast_net.py:22-33): X (F*J, C) -> out (F*J, 2C)
static int run_block(gast_handle* h, cudaStream_t st, BlockConsts& b, const float* X, long long F,
                     const BlockBufs& w, float* out) {
  const int C = b.C;
  if (run_local(h, st, b, X, F, w, w.L, GAST_KIND_BLOCK)) return 1;
  if (run_global(h, st, b, X, F, w, w.Gl, GAST_KIND_BLOCK)) return 1;
  GemmP p;
  gemm_defaults_flat(p, h, F);
  p.nseg = 3;
  p.seg[0] = seg_flat(X, C, C); p.seg[1] = seg_flat(w.L, C, C); p.seg[2] = seg_flat(w.Gl, C, C);
  p.W = b.Wbc; p.ldw = 3 * C; p.N = 2 * C; p.out = out; p.ld_out = 2 * C; p.bias = b.bbc; p.relu = 1;
  return launch_gemm(h, st, EPI_PLAIN, p, &b.tc_bc);
}

// expand (gast_net.py:163-164): rows output positions, windows of x (clips of T frames, stride `stride`) -> out (rows, C)
static int launch_expand(gast_handle* h, cudaStream_t st, const float* x, float* out, long long rows, int T, int T0,
                         int stride) {
  const gast_cfg& c = h->cfg;
  const int k0 = c.filter_widths[0], Fin = c.in_features;
  if (rows >= 0x7fffffffLL) return fail("expand: more than 2^31 positions in one call");
  if (k0 * Fin > EXP_MAXKF) return fail("expand: filter_width*in_features > %d unsupported", EXP_MAXKF);
  return with_types(h, [&](auto io, auto act) {
    using Io = typename decltype(io)::type;
    using Act = typename decltype(act)::type;
    auto fill = [&](gast_kernel_audit& d) {
      d.kind = KA_EXPAND; d.variant = k0 * Fin <= 6 ? 6 : EXP_MAXKF;
      d.in_type = elem_dtype<Io>; d.out_type = elem_dtype<Act>; d.x = x; d.We = h->We; d.be = h->be; d.out = out;
      d.rows = rows; d.K = c.channels; d.ld = c.channels; d.J = c.num_joints; d.T = T; d.T0 = T0; d.stride = stride;
      d.taps = k0; d.Fin = Fin;
    };
    return kernel_audited(h, st, LK_EXPAND, fill, [&] {
      const dim3 grid(cdiv(rows, EXS_ROWS), cdiv(c.channels, EXS_CHUNK));
      const auto kernel = k0 * Fin <= 6 ? expand_rows_kernel<6, Io, Act> : expand_rows_kernel<EXP_MAXKF, Io, Act>;
      kernel<<<grid, EXS_THREADS, 0, st>>>(reinterpret_cast<const Io*>(x), h->We, h->be, reinterpret_cast<Act*>(out),
                                           rows, c.num_joints, T, T0, stride, k0, Fin, c.channels);
      return 0;
    });
  });
}

// temporal stage on F frames: conv over the taps of `taps` + BN + ReLU into tmp, then 1x1 conv + BN + ReLU (+Dropout =
// identity in eval) + the residual rows res_map of `res` into out (gast_net.py:170,173-174 / :243,247)
static int run_stage(gast_handle* h, cudaStream_t st, const StageConsts& s, long long F, const ASeg& taps,
                     const float* Wt, const TcWeights* tc_t, float* tmp, const float* res, RowMap res_map, float* out) {
  const int Cw = s.Cw;
  GemmP p;
  gemm_defaults(p, h, F);
  p.nseg = 1; p.seg[0] = taps;
  p.W = Wt; p.ldw = taps.K; p.N = Cw; p.out = tmp; p.ld_out = Cw; p.bias = s.bt; p.relu = 1;
  if (launch_gemm(h, st, EPI_PLAIN, p, tc_t)) return 1;
  gemm_defaults(p, h, F);
  p.nseg = 1; p.seg[0] = seg_flat(tmp, Cw, Cw);
  p.W = s.W1; p.ldw = Cw; p.N = Cw; p.out = out; p.ld_out = Cw; p.bias = s.b1; p.relu = 1;
  p.res = res; p.res_ld = Cw; p.res_map = res_map;
  return launch_gemm(h, st, EPI_PLAIN, p, &s.tc_1);
}

// shrink (gast_net.py:99): X (rows, C << L) -> y (rows, 3); with a target also the mpjpe of y into *loss, its block
// partials and ticket in `scratch` (LOSS_SCRATCH_FLOATS of the call's workspace, ModelBufs::loss)
static int launch_shrink(gast_handle* h, cudaStream_t st, const float* X, float* y, long long rows, const float* target,
                         float* loss, float* scratch = nullptr) {
  Lookup Lk{h};
  const int Cl = h->cfg.channels << h->cfg.num_stages;
  const float* ws = Lk.get("shrink.weight", (int64_t)3 * Cl);
  if (!Lk.ok) return 1;
  if (target && !scratch) return fail("gast_forward_mpjpe: no loss scratch in the workspace");
  // a fresh workspace is not zeroed: clear the ticket on the call's stream (a captured graph replays this memset too)
  if (target) CUDA_OK(cudaMemsetAsync(scratch + 2 * SHL_MAXBLOCKS, 0, sizeof(unsigned), st));
  return with_types(h, [&](auto io, auto act) {
    using Io = typename decltype(io)::type;
    using Act = typename decltype(act)::type;
    auto fill = [&](gast_kernel_audit& d) {
      d.kind = target ? KA_SHRINK_MPJPE : KA_SHRINK;
      d.in_type = elem_dtype<Act>; d.out_type = elem_dtype<Io>; d.x = X; d.Ws = ws; d.target = target;
      d.loss = loss; d.out = y; d.rows = rows; d.K = Cl; d.ld = Cl;
    };
    return kernel_audited(h, st, LK_SHRINK, fill, [&] {
      const Act* x = reinterpret_cast<const Act*>(X);
      if (target) {   // y, target and the loss are float32 (a half model refuses the mpjpe forward)
        double* partial = reinterpret_cast<double*>(scratch);
        unsigned* ticket = reinterpret_cast<unsigned*>(scratch + 2 * SHL_MAXBLOCKS);
        const unsigned nb = (unsigned)std::min<long long>(SHL_MAXBLOCKS, (rows + 7) / 8);
        shrink_mpjpe_kernel<<<nb, 256, 0, st>>>(x, Cl, ws, y, rows, Cl, target, partial, ticket, loss);
      } else {
        shrink_kernel<<<cdiv(rows * 32, 256), 256, 0, st>>>(x, Cl, ws, reinterpret_cast<Io*>(y), rows, Cl);
      }
      return 0;
    });
  });
}

// In a half forward (gast_set_activation_dtype) and at the fp16 precision (with_types) every buffer but bb.AB holds fp16:
// the pointers are typed float and the launches reinterpret them.
struct ModelBufs {
  float* act[2];
  float* tmp;
  BlockBufs bb;
  float* loss;   // gast_forward_mpjpe's SHL_MAXBLOCKS double partials and ticket: in the workspace, so that calls on
                 // distinct workspaces never share them
};

constexpr size_t LOSS_SCRATCH_FLOATS = 2 * SHL_MAXBLOCKS + 4;

static int plan_model(const gast_handle* h, int B, int T, int strided_now, Arena& a, ModelBufs* mb, Geometry* g) {
  if (geometry(h, T, strided_now, g)) return 1;
  a.esize = act_esize(h);
  const int J = h->cfg.num_joints, C = h->cfg.channels, L = h->cfg.num_stages;
  // max over layers
  size_t act = 0, tmp = 0, xy = 0, l = 0, ab = 0;
  long long rows = (long long)B * g->T0 * J;
  for (int i = 0; i < L; ++i) {
    const int Cw = C << i;
    if (i > 0) {
      rows = (long long)B * g->stages[i - 1].Tout * J;
      tmp = std::max(tmp, (size_t)rows * Cw);
    }
    act = std::max(act, (size_t)rows * 2 * Cw);
    xy = std::max(xy, (size_t)rows * 2 * Cw);
    l = std::max(l, (size_t)rows * Cw);
    ab = std::max(ab, (size_t)rows * 8);
  }
  mb->act[0] = a.take(act); mb->act[1] = a.take(act);
  mb->tmp = a.take(tmp);
  mb->bb.XY = a.take(xy); mb->bb.L = a.take(l); mb->bb.AB = a.take32(ab); mb->bb.Y = a.take(l); mb->bb.Gl = a.take(l);
  mb->loss = a.take32(LOSS_SCRATCH_FLOATS);
  return 0;
}

extern "C" size_t gast_workspace_bytes(const gast_t* h, int32_t B, int32_t T, int32_t strided_now) {
  if (!h) return 0;
  Arena a{nullptr, 0, 0, true};
  if (h->cfg.kind == GAST_KIND_MODEL) {
    ModelBufs mb; Geometry g;
    if (plan_model(h, B, T, strided_now, a, &mb, &g)) return 0;
  } else {
    BlockBufs bb;
    const BlockConsts& b = h->blocks[0];
    block_bufs(a, (long long)B * h->cfg.num_joints, b.C, b.Cout, b.heads ? b.heads : 4, b.Cg ? b.Cg : b.C / 4, &bb);
  }
  return a.off + 256;
}

// The start of every model and streaming call once its own checks passed: a null or short workspace is refused, the
// handle's device is made current and the launch counters and timing events restart for this call.  A backward
// (restart_counts false) continues the counts of its training forward instead.
static int call_begin(gast_handle* h, const char* who, size_t need, void* workspace, size_t workspace_bytes,
                      bool restart_counts = true) {
  if (!workspace || workspace_bytes < need)
    return fail("%s: workspace too small (%zu < %zu bytes)", who, workspace_bytes, need);
  CUDA_OK(cudaSetDevice(h->cfg.device));
  if (restart_counts) {
    h->launches = h->tc_launches = h->wgrad_tc_launches = 0;
    h->ev_used = 0;
    h->ev_kind.clear();
  }
  return 0;
}

// The launches of a MODEL-kind forward on the workspace carved by `a` (the caller has checked its size)
static int model_forward(gast_handle* h, cudaStream_t st, const float* x, float* y, int B, int T, int strided_now, Arena a,
                         const float* target, float* loss) {
  const int J = h->cfg.num_joints;
  ModelBufs mb; Geometry g;
  if (plan_model(h, B, T, strided_now, a, &mb, &g)) return 1;
  // expand (gast_net.py:163-164) + first GraphAttentionBlock
  long long F = (long long)B * g.T0;
  if (launch_expand(h, st, x, mb.act[0], F * J, T, g.T0, g.s0)) return 1;
  if (run_block(h, st, h->blocks[0], mb.act[0], F, mb.bb, mb.act[1])) return 1;
  int cur = 1;
  for (int i = 1; i < h->cfg.num_stages; ++i) {
    StageConsts& s = h->stages[i - 1];
    const StageGeo& sg = g.stages[i - 1];
    const int Cw = s.Cw;
    const long long Fn = (long long)B * sg.Tout;
    const float* xin = mb.act[cur];
    const ASeg taps = seg_taps(xin, Cw, Cw, sg.taps, (long long)sg.dil * J * Cw, sg.tapmap);
    if (run_stage(h, st, s, Fn, taps, s.Wt, &s.tc_t, mb.tmp, xin, sg.resmap, mb.act[cur ^ 1])) return 1;
    cur ^= 1;
    if (run_block(h, st, h->blocks[i], mb.act[cur], Fn, mb.bb, mb.act[cur ^ 1])) return 1;
    cur ^= 1;
    F = Fn;
  }
  // output is already (B, T_out, J, 3)
  if (launch_shrink(h, st, mb.act[cur], y, F * J, target, loss, mb.loss)) return 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

static int forward_impl(gast_t* h, const float* x, float* y, int32_t B, int32_t T, int32_t strided_now,
                        void* workspace, size_t workspace_bytes, void* stream, const float* target, float* loss) {
  if (!h) return fail("gast_forward: null handle");
  if (!h->prepared) return fail("gast_forward: gast_prepare() has not run since the last gast_bind()");
  if (B <= 0 || T <= 0) return fail("gast_forward: empty batch (B=%d T=%d)", B, T);
  const int kind = h->cfg.kind;
  if (kind != GAST_KIND_MODEL && T != 1) return fail("gast_forward: module kinds take T == 1 (frames in B)");
  const size_t need = gast_workspace_bytes(h, B, T, strided_now);
  if (need == 0) return 1;
  if (call_begin(h, "gast_forward", need, workspace, workspace_bytes)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Arena a = workspace_arena(workspace, workspace_bytes);
  const int J = h->cfg.num_joints;

  if (kind != GAST_KIND_MODEL) {
    BlockConsts& b = h->blocks[0];
    BlockBufs bb;
    block_bufs(a, (long long)B * J, b.C, b.Cout, b.heads ? b.heads : 4, b.Cg ? b.Cg : b.C / 4, &bb);
    int rc = 0;
    if (kind == GAST_KIND_BLOCK) rc = run_block(h, st, b, x, B, bb, y);
    else if (kind == GAST_KIND_LOCAL || kind == GAST_KIND_SEMCH) rc = run_local(h, st, b, x, B, bb, y, kind);
    else rc = run_global(h, st, b, x, B, bb, y, kind);
    if (rc) return 1;
    CUDA_OK(cudaGetLastError());
    return 0;
  }
  return model_forward(h, st, x, y, B, T, strided_now, a, target, loss);
}

extern "C" int gast_forward(gast_t* h, const float* x, float* y, int32_t B, int32_t T, int32_t strided_now,
                            void* workspace, size_t workspace_bytes, void* stream) {
  return forward_impl(h, x, y, B, T, strided_now, workspace, workspace_bytes, stream, nullptr, nullptr);
}

// forward + mpjpe of the prediction against `target` (B, T_out, J, 3) in one call: the caller-side pair
// `predicted = model(x); error = mpjpe(predicted, target)` of main.py:evaluate / train with the loss taken in the shrink
// kernel's epilogue (SURVEY §8f N2)
extern "C" int gast_forward_mpjpe(gast_t* h, const float* x, const float* target, float* y, float* loss, int32_t B, int32_t T,
                                  int32_t strided_now, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h) return fail("gast_forward_mpjpe: null handle");
  if (h->cfg.kind != GAST_KIND_MODEL) return fail("gast_forward_mpjpe: only the MODEL kind has a shrink layer");
  if (!target || !loss) return fail("gast_forward_mpjpe: target and loss must be device pointers");
  if (half_check(h, "gast_forward_mpjpe")) return 1;
  return forward_impl(h, x, y, B, T, strided_now, workspace, workspace_bytes, stream, target, loss);
}

#include "stream.cuh"

// ------------------------------------------------------------------------------------------
// test-time augmentation around the forward (SURVEY.md §8f N1)
// ------------------------------------------------------------------------------------------
static int make_perm(int J, int n, const int32_t* left, const int32_t* right, JointPerm* p) {
  if (J < 1 || J > 32) return fail("tta: J out of range");
  for (int j = 0; j < 32; ++j) p->p[j] = (unsigned char)j;
  for (int k = 0; k < n; ++k) {
    if (left[k] < 0 || left[k] >= J || right[k] < 0 || right[k] >= J) return fail("tta: joint index out of range");
    p->p[left[k]] = (unsigned char)right[k];
    p->p[right[k]] = (unsigned char)left[k];
  }
  return 0;
}

extern "C" int gast_tta_prepare(const float* seq, float* out, int32_t T, int32_t J, int32_t F, int32_t pad,
                                int32_t causal_shift, int32_t n_sym, const int32_t* kps_left, const int32_t* kps_right,
                                void* stream) {
  if (T <= 0 || F <= 0 || pad < 0 || causal_shift < 0 || causal_shift > pad) return fail("gast_tta_prepare: bad arguments");
  JointPerm perm;
  if (make_perm(J, n_sym, kps_left, kps_right, &perm)) return 1;
  const long long n = (long long)(T + 2 * pad) * J * F;
  tta_prepare_kernel<<<cdiv(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      seq, out, T, J, F, pad + causal_shift, pad - causal_shift, perm);
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_tta_merge(const float* pred, float* out, int32_t T, int32_t J, int32_t n_sym,
                              const int32_t* joints_left, const int32_t* joints_right, void* stream) {
  if (T <= 0) return fail("gast_tta_merge: bad arguments");
  JointPerm perm;
  if (make_perm(J, n_sym, joints_left, joints_right, &perm)) return 1;
  const long long n = (long long)T * J * 3;
  tta_merge_kernel<<<cdiv(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pred, out, T, J, perm);
  CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------
// training (SURVEY.md §8 row a12)
// ------------------------------------------------------------------------------------------
#include "train.cuh"

extern "C" int gast_bind_grads(gast_t* h, int32_t n, const char* const* keys, void* const* ptrs, const int64_t* numel) {
  if (!h) return fail("gast_bind_grads: null handle");
  for (int i = 0; i < n; ++i) h->grads[keys[i]] = Binding{ptrs[i], numel[i]};
  return 0;
}

// The inference precision alone does not reach training: a handle at inference TF32 trains and differentiates only
// once the training precision is TF32 too (gast_set_train_precision), and nothing falls back silently
static int precision_check(gast_handle* h, const char* what) {
  if (half_check(h, what)) return 1;
  if (h->precision != 0 && h->train_precision == 0)
    return fail("%s: reduced precision is inference-only; call gast_set_precision(h, 0) before training or "
                "differentiating (precision is %d)", what, h->precision);
  return 0;
}

static int train_check(gast_handle* h, const char* what) {
  if (h->cfg.kind != GAST_KIND_MODEL) return fail("training is implemented for the MODEL kind only");
  return precision_check(h, what);
}

static Arena sizing_arena(size_t off = 0) { return Arena{nullptr, 0, off, true}; }

// The workspace of a training forward + backward of the mode `ts` describes, by their sizing pass in c; 0 on error.
// c keeps the pass's lookups for the caller to refuse on.
static size_t train_sizing(TCtx& c, int B, int T, TrainState ts) {
  if (train_forward(c.h, c, ts, nullptr, nullptr, B, T) || train_backward(c.h, c, ts, nullptr, nullptr)) return 0;
  return c.a.off + 512;
}

extern "C" size_t gast_train_workspace_bytes(gast_t* h, int32_t B, int32_t T, float dropout_p) {
  if (!h || train_check(h, "gast_train_workspace_bytes")) return 0;
  TrainState ts;
  ts.drop_p = dropout_p;
  TCtx c(h, nullptr, sizing_arena(), true);
  return train_sizing(c, B, T, ts);
}

extern "C" int gast_forward_train(gast_t* h, const float* x, float* y, int32_t B, int32_t T, float dropout_p,
                                  uint64_t seed, void* workspace, size_t workspace_bytes, void* stream) {
  if (!h) return fail("gast_forward_train: null handle");
  if (train_check(h, "gast_forward_train")) return 1;
  if (B <= 0 || T <= 0) return fail("gast_forward_train: empty batch (B=%d T=%d)", B, T);
  if (!x || !y) return fail("gast_forward_train: x and y must be device pointers");
  if (dropout_p < 0.f || dropout_p >= 1.f) return fail("gast_forward_train: dropout_p out of range");
  TrainState sized;
  sized.drop_p = dropout_p;
  TCtx dry(h, nullptr, sizing_arena(), true);
  const size_t need = train_sizing(dry, B, T, sized);
  // gradient buffers are only read by the backward, which checks them itself
  if (need == 0 || dry.refuse(false)) return 1;
  if (call_begin(h, "gast_forward_train", need, workspace, workspace_bytes)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TCtx c(h, st, workspace_arena(workspace, workspace_bytes), true);
  for (size_t i = 0; i < h->trains.size(); ++i)      // a workspace reused by the caller: its old state is dead
    if (h->trains[i].first == workspace) { h->trains.erase(h->trains.begin() + i); break; }
  if (h->trains.size() >= GAST_MAX_PENDING_TRAIN) h->trains.erase(h->trains.begin());   // forwards never differentiated
  h->trains.emplace_back(workspace, TrainState());
  TrainState& ts = h->trains.back().second;
  ts.drop_p = dropout_p;
  ts.seed = seed;
  ts.workspace_bytes = need;
  if (train_forward(h, c, ts, x, y, B, T)) { h->trains.pop_back(); return 1; }
  ts.arena_off = c.a.off;
  ts.valid = true;
  if (h->dropout_state && dropout_p > 0.f) dropout_bump_kernel<<<1, 1, 0, st>>>(h->dropout_state);
  h->prepared = false;      // running statistics changed: eval constants are stale
  CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int gast_set_dropout_state(gast_t* h, void* dev_u64) {
  if (!h) return fail("gast_set_dropout_state: null handle");
  h->dropout_state = reinterpret_cast<unsigned long long*>(dev_u64);
  return 0;
}

extern "C" int gast_backward(gast_t* h, const float* dy, void* workspace, size_t workspace_bytes, void* stream) {
  return gast_backward_input(h, dy, nullptr, 1, workspace, workspace_bytes, stream);
}

extern "C" int gast_backward_input(gast_t* h, const float* dy, float* dx, int32_t param_grads, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  if (!h) return fail("gast_backward: null handle");
  if (precision_check(h, "gast_backward")) return 1;
  if (!dy) return fail("gast_backward: dy must be a device pointer");
  if (!dx && !param_grads) return fail("gast_backward_input: neither dx nor parameter gradients requested");
  size_t ti = h->trains.size();
  for (size_t i = 0; i < h->trains.size(); ++i)
    if (h->trains[i].first == workspace) ti = i;
  if (ti == h->trains.size() || !h->trains[ti].second.valid)
    return fail("gast_backward: no training forward is saved in this workspace (already differentiated, "
                "or more than %d forwards were outstanding)", GAST_MAX_PENDING_TRAIN);
  if (call_begin(h, "gast_backward", h->trains[ti].second.workspace_bytes, workspace, workspace_bytes, false)) return 1;
  TrainState ts = h->trains[ti].second;
  TCtx dry(h, nullptr, sizing_arena(ts.arena_off), param_grads != 0);
  if (train_backward(h, dry, ts, nullptr, nullptr) || dry.refuse(true)) return 1;   // the saved forward stays
  h->trains.erase(h->trains.begin() + ti);
  TCtx c(h, reinterpret_cast<cudaStream_t>(stream), workspace_arena(workspace, workspace_bytes, ts.arena_off),
         param_grads != 0);
  c.tc_slot = 1024;                         // the backward's GEMMs follow the forward's in the operand-copy table
  if (train_backward(h, c, ts, dy, dx)) return 1;
  CUDA_OK(cudaGetLastError());
  return 0;
}

#include "chunked.cuh"

// Timing of the debug entries: `launch` once, then `reps` more times between two events on `st`; waits for the stream
// and, when all of it succeeded and reps > 0, stores the ms per rep in *ms_out.  Returns 0, the first failing launch's
// code or the stream's error.
template <class Launch>
static int timed_reps(cudaStream_t st, int reps, float* ms_out, Launch launch) {
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  int rc = (int)cudaEventCreate(&e0);
  if (!rc) rc = (int)cudaEventCreate(&e1);
  if (!rc) rc = launch();
  if (!rc && reps > 0) {
    cudaEventRecord(e0, st);
    for (int i = 0; i < reps && !rc; ++i) rc = launch();
    cudaEventRecord(e1, st);
  }
  const cudaError_t e = cudaStreamSynchronize(st);
  if (!rc) rc = (int)e;
  if (!rc && reps > 0 && ms_out) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    *ms_out = ms / reps;
  }
  if (e0) cudaEventDestroy(e0);
  if (e1) cudaEventDestroy(e1);
  return rc;
}

// ------------------------------------------------------------------------------------------
// debug / probe entry: out[M,N] = A[M,K] . W[N,K]^T on a chosen GEMM core (test infrastructure
// for the numerics of the tensor-core path; not used by the forward).  tc_mode: the tensor-core core's precision
// (0 fp32-grade as inference runs it, three fp16 products on scaled operands; 1 single-pass TF32; 3 fp32-grade as
// training runs it, three TF32 products; 16 the half form, on fp16 A and out).
// ------------------------------------------------------------------------------------------
extern "C" int gast_debug_gemm(const float* A, const float* W, float* out, int32_t M, int32_t N, int32_t K,
                               int32_t core, int32_t tc_mode, int32_t reps, float* ms_out, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (M <= 0 || N <= 0 || K <= 0 || N % 4 || K % 4) return fail("gast_debug_gemm: bad shape");
  if (core < 0 || core > 1 || (tc_mode != 0 && tc_mode != 1 && tc_mode != 3 && tc_mode != 16) ||
      (core == 1 && tc_mode != 0))
    return fail("gast_debug_gemm: core must be 0 (tensor cores, tc_mode 0 = F16X3, 1 = TF32, 3 = 3xTF32 or 16 = the "
                "half form) or 1 (FFMA, tc_mode 0)");
  GemmP p;
  gemm_flat(p, M);
  p.nseg = 1; p.seg[0] = seg_flat(A, K, K);
  p.W = W; p.ldw = K; p.N = N; p.out = out; p.ld_out = N;
  int rc = 0;
  std::vector<void*> owned;
  TcWeights t;
  if (core == 0) {
    rc = tc_prepare_weights(t, W, N, K, st, &owned, tc_mode != 3);   // 3xTF32 runs on training's tf32 copies
    if (rc || !t.ready || !(tc_mode == 16 ? tc_supported_h(p, EPI_PLAIN, t) : tc_supported(p, EPI_PLAIN, t))) {
      for (void* q : owned) cudaFree(q);
      return fail("gast_debug_gemm: shape not supported by the tensor-core core (rc=%d)", rc);
    }
  } else {
    cudaFuncSetAttribute((const void*)gemm_ffma_kernel<EPI_PLAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024);
  }
  rc = timed_reps(st, reps, ms_out, [&]() -> int {
    if (core == 0) return tc_launch(st, EPI_PLAIN, p, t, tc_mode == 16 ? TC_F16 : tc_prec(t, tc_mode == 1));
    dim3 grid(cdiv(M, 128), cdiv(N, FF_BN));
    gemm_ffma_kernel<EPI_PLAIN><<<grid, FF_THREADS, ffma_smem_bytes(EPI_PLAIN, 1, 128, 1), st>>>(p);
    return (int)cudaGetLastError();
  });
  for (void* q : owned) cudaFree(q);
  if (rc) return fail("gast_debug_gemm: %s", cudaGetErrorString((cudaError_t)rc));
  return 0;
}

// ------------------------------------------------------------------------------------------
// debug / probe entry: dW[N,K] = dZ[M,N]^T . A[M,K] (dense leading dimensions) as the training backward computes a
// weight gradient: dense_tn's row splits on this device, one kernel over them, the fixed-order reduction.  core 1:
// wgrad_tn_kernel (FFMA, exact fp32; tc_mode 0).  core 0 with tc_mode 1: the kernel the TF32 training precision
// picks, wgrad_tc_kernel where it takes the shape and wgrad_tn_kernel elsewhere.  There is no fp32-grade tensor-core
// weight gradient, so core 0 with tc_mode 0 is refused.  reps > 0 times reps more runs of both kernels into *ms_out
// (ms per run).
// ------------------------------------------------------------------------------------------
extern "C" int gast_debug_wgrad(const float* dZ, const float* A, float* dW, int32_t M, int32_t N, int32_t K,
                                int32_t core, int32_t tc_mode, int32_t reps, float* ms_out, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (M <= 0 || N <= 0 || K <= 0) return fail("gast_debug_wgrad: bad shape");
  if (core == 0 && tc_mode == 0)
    return fail("gast_debug_wgrad: there is no fp32-grade tensor-core weight gradient (core 0 needs tc_mode 1)");
  if (core < 0 || core > 1 || tc_mode < 0 || tc_mode > 1 || (core == 1 && tc_mode != 0))
    return fail("gast_debug_wgrad: core must be 0 (tensor cores, tc_mode 1 = TF32) or 1 (FFMA, tc_mode 0)");
  int dev = 0;
  CUDA_OK(cudaGetDevice(&dev));
  int sms = 0;
  CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  long long S, rps;
  wgrad_split(M, N, K, sms, &S, &rps);
  float* part = nullptr;
  CUDA_OK(cudaMalloc(&part, sizeof(float) * (size_t)S * N * K));
  bool on_tc = false;
  const int rc = timed_reps(st, reps, ms_out,
                            [&]() { return wgrad_run(st, dZ, N, A, K, M, N, K, S, rps, part, dW, K, core == 0, &on_tc); });
  cudaFree(part);
  if (rc) return fail("gast_debug_wgrad: %s", cudaGetErrorString((cudaError_t)rc));
  return 0;
}

// ------------------------------------------------------------------------------------------
// callers / data formats either side of the forward (SURVEY.md §8f N1-N3)
// ------------------------------------------------------------------------------------------
#include "pipeline.cuh"

// ------------------------------------------------------------------------------------------
// the reconstruction's animation frames (DESIGN.md §8.5)
// ------------------------------------------------------------------------------------------
#include "render.cuh"

// ------------------------------------------------------------------------------------------
// the 2D pose net's person crops and heatmap decode (DESIGN.md §8.6)
// ------------------------------------------------------------------------------------------
#include "keypoints2d.cuh"

// ------------------------------------------------------------------------------------------
// the person detector's letterbox and post-processing (DESIGN.md §8.7)
// ------------------------------------------------------------------------------------------
#include "detect.cuh"

// ------------------------------------------------------------------------------------------
// the SORT tracker between the detector and the 2D pose net (DESIGN.md §8.8)
// ------------------------------------------------------------------------------------------
#include "track.cuh"

// ------------------------------------------------------------------------------------------
// SORT's tracks to the 2D pose net's crop records (DESIGN.md §8.9)
// ------------------------------------------------------------------------------------------
#include "records.cuh"
#include "live.cuh"
