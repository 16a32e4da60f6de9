/*
 * gast_b200.h -- C ABI of the H100-native GAST-Net 2D->3D lifting path (libgast_b200.so).
 *
 * The reference (fabro66/GAST-Net-3DPoseEstimation) is pure Python and has no FFI for this
 * path; its "plugin boundary" is the Python class API of model/gast_net.py.  This header is
 * the C boundary underneath our drop-in classes: plain pointers and sizes, no torch types.
 * Each entry point cites the reference interface it stands in for.
 *
 * Ownership: the caller owns ALL device memory that crosses this boundary (parameters,
 * buffers, gradients, inputs, outputs, workspace).  A handle owns only small derived
 * constants (folded/packed weights) that gast_prepare() recomputes.  Nothing here
 * synchronises the device or allocates on the forward path; all work is enqueued on the
 * caller's stream.  Every call returns 0 on success, non-zero on error with a message in
 * gast_last_error() (thread-local).  Nothing throws or aborts.
 */
#ifndef GAST_B200_H
#define GAST_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gast_handle gast_t;

/* What a handle computes.  MODEL is the product; the others are the reference's
 * sub-modules, exposed so that parity can be tested module by module. */
enum gast_kind {
  GAST_KIND_MODEL = 0,       /* SpatioTemporalModel / ...Optimized1f   model/gast_net.py:107,180 */
  GAST_KIND_BLOCK = 1,       /* GraphAttentionBlock                    model/gast_net.py:8-33    */
  GAST_KIND_LOCAL = 2,       /* LocalGraph                             model/local_attention.py:59-151 */
  GAST_KIND_MGLOBAL = 3,     /* MultiGlobalGraph                       model/global_attention.py:85-130 */
  GAST_KIND_SEMCH = 4,       /* SemCHGraphConv / SemGraphConv          model/local_attention.py:10-56, model/sem_graph_conv.py:10-55 */
  GAST_KIND_GLOBAL_HEAD = 5  /* GlobalGraph                            model/global_attention.py:7-82 */
};

#define GAST_MAX_STAGES 8

/* Mirrors the constructor arguments of SpatioTemporalModel(adj, num_joints_in, in_features,
 * num_joints_out, filter_widths, causal, dropout, channels, dense) (model/gast_net.py:113-114)
 * and SpatioTemporalModelOptimized1f(...) (:191-192).  The adjacency enters as the two
 * LocalGraph masks (model/local_attention.py:92-114) in row-major nonzero order, which is the
 * order the learnable `e` is scattered in (:25,:41). */
typedef struct gast_cfg {
  int32_t kind;                          /* enum gast_kind */
  int32_t num_joints;                    /* J: 15, 16, 17 or 19 */
  int32_t in_features;                   /* 2 (MODEL only) */
  int32_t channels;                      /* MODEL: `channels`; other kinds: input width C */
  int32_t channels_out;                  /* SEMCH: out_features; GLOBAL_HEAD: inter_channels; else 0 */
  int32_t num_stages;                    /* len(filter_widths) (MODEL only) */
  int32_t filter_widths[GAST_MAX_STAGES];
  int32_t causal;
  int32_t dense;                         /* SpatioTemporalModel(dense=True) ablation */
  int32_t strided;                       /* 1 = Optimized1f schedule, 0 = dilated */
  int32_t heads;                         /* MGLOBAL/GLOBAL_HEAD: number of heads (BLOCK/MODEL: 4) */
  int32_t semch_shared_e;                /* SEMCH: 1 = one `e` row shared by all channels (sem_graph_conv.py) */
  int32_t semch_bias;                    /* SEMCH: 1 = has bias */
  int32_t sym_nnz, con_nnz;              /* nonzeros of the two masks (SEMCH uses `sym` only) */
  const int32_t* sym_rows; const int32_t* sym_cols;   /* host arrays, row-major nonzero order */
  const int32_t* con_rows; const int32_t* con_cols;
  int32_t device;                        /* CUDA device ordinal */
} gast_cfg;

/* nn.Module construction (gast_net.py:113-157).  Copies cfg (incl. the mask arrays). */
int gast_create(gast_t** out, const gast_cfg* cfg);
void gast_destroy(gast_t* h);

/* Borrow the caller's parameter / buffer storage by state_dict key (SURVEY.md 8b lists the
 * keys; they are exactly `module.state_dict().keys()` of the reference classes).  Pointers
 * are device pointers to contiguous fp32 (int64 for num_batches_tracked, ignored).  No copy:
 * optimiser updates are seen after the next gast_prepare().  Stands in for
 * nn.Module.load_state_dict / .parameters() (main.py:193,207-208). */
int gast_bind(gast_t* h, int32_t n, const char* const* keys, void* const* dev_ptrs,
              const int64_t* numel);

/* Recompute the eval-mode derived constants from the bound parameters: BN folded into the
 * adjacent conv, softmaxed per-channel adjacencies, packed SemCH weights, collapsed
 * theta/phi vectors.  Call after binding and after every parameter change (the Python shim
 * tracks tensor versions).  Enqueued on `stream` (a cudaStream_t). */
int gast_prepare(gast_t* h, void* stream);

/* Output frames for an input of T frames: T - rf + 1 (dilated) or the strided count
 * (gast_net.py:62-69,159-177,236-251).  `strided_now` = schedule actually used. Returns <0 on error. */
int32_t gast_out_frames(const gast_t* h, int32_t T, int32_t strided_now);
int32_t gast_receptive_field(const gast_t* h);

/* Bytes of caller-provided scratch gast_forward needs for a (B,T) batch. */
size_t gast_workspace_bytes(const gast_t* h, int32_t B, int32_t T, int32_t strided_now);

/* forward(x) (gast_net.py:84-104), eval mode.
 *   MODEL:  x (B,T,J,in_features) fp32 -> y (B,T_out,J,3) fp32, both contiguous.
 *           strided_now: 0 = dilated schedule (any T >= rf), 1 = strided schedule
 *           (T a multiple of the receptive field pattern, as Optimized1f requires).
 *   other kinds: x is (B frames, J, C) with T == 1; y is (B, J, C_out)
 *           (BLOCK: C_out = 2C, channels-last).
 * All work is enqueued on `stream`. */
int gast_forward(gast_t* h, const float* x, float* y, int32_t B, int32_t T,
                 int32_t strided_now, void* workspace, size_t workspace_bytes, void* stream);

/* forward + mpjpe in one call: the caller-side pair `predicted = model(x); error = mpjpe(predicted, target)` of
 * main.py:evaluate (main.py:270-300) and of the training loop's validation pass, with the loss of common/loss.py:5-11
 * taken in the shrink kernel's epilogue (no second pass over the prediction).  MODEL kind only.
 *   target (B,T_out,J,3) fp32 device; y as gast_forward; *loss (device float) = mean over B*T_out*J joints of
 *   ||y - target||_2.  Block partial sums are double and are added in a fixed order: the loss is reproducible run to run. */
int gast_forward_mpjpe(gast_t* h, const float* x, const float* target, float* y, float* loss, int32_t B, int32_t T,
                       int32_t strided_now, void* workspace, size_t workspace_bytes, void* stream);

/* Launch counters.  Every forward-type call (gast_forward, gast_forward_mpjpe, gast_forward_train,
 * gast_eval_backward and each gast_stream_* push or peek) starts this count, the two below and the timing events at
 * zero once its checks pass; gast_backward(_input) continues the counts of its training forward, so after a training
 * step they cover the whole step.
 * gast_last_launch_count: number of kernels the last such call enqueued (for bench.py's gpu_launches). */
int32_t gast_last_launch_count(const gast_t* h);

/* Number of those that ran on the tensor-core (wgmma) GEMM core, in either precision (gast_set_precision). */
int32_t gast_last_tc_launch_count(const gast_t* h);

/* Per-launch device timing for the roofline report: when on, gast_forward brackets every
 * kernel launch with a CUDA event pair on the caller's stream; gast_get_timings waits for
 * them and returns up to max_n (milliseconds, kind) pairs of the last forward.  kinds:
 * 0 expand, 1-3 FFMA GEMM (plain/SemCH/global epilogue), 4 theta/phi row-dot, 5 shrink,
 * 6-8 tensor-core GEMM (plain/SemCH/global), 9 attention mix of MultiGlobalGraph as its own kernel. */
int gast_set_timing(gast_t* h, int32_t on);
int32_t gast_get_timings(gast_t* h, int32_t max_n, float* ms, int32_t* kinds);

/* GEMM core selection for A/B checks on the GPU: 0 = auto (tensor cores where the shape
 * allows; fp32-grade or single-pass TF32 as gast_set_precision says), 1 = force the FP32 FFMA core (fp32 in either
 * precision; refused at the fp16 precision and in half, which run on the tensor cores only).  Not a fallback switch:
 * both are CUDA paths. */
int gast_set_gemm_core(gast_t* h, int32_t core);

/* Arithmetic of the GEMMs the tensor-core core runs, for every handle kind and for gast_forward,
 * gast_forward_mpjpe and the gast_stream_push* calls:
 *   0 = fp32-grade (default), within ~1e-7 relative of an fp32 GEMM: three fp16 products on operands scaled by
 *       exact powers of two (per weight matrix, and per row and 32-K stage of A), fp32's full range; training and
 *       every gradient run the equally precise 3xTF32.
 *   1 = TF32: tf32(A) . tf32(W) with fp32 accumulation, one tensor-core product per multiply-add.  Operands are
 *       rounded to 10 mantissa bits (round to nearest, ties away), so outputs move by ~1e-3 relative
 *       (DESIGN.md §4.1).  Inference only: gast_forward_train, gast_backward(_input), gast_eval_backward and their
 *       workspace queries fail while it is set, unless the training precision is TF32 too (gast_set_train_precision).
 *   16 = fp16 (GAST_PRECISION_F16), MODEL kind only: the arithmetic and activation storage of the half form
 *       (gast_set_activation_dtype(h, GAST_F16)) behind float32 x, y and parameters.  Every activation in the
 *       workspace is fp16 (the attention row dots stay fp32); every GEMM is one fp16 product per multiply-add on
 *       fp16(W 2^s_W) with fp32 accumulation; expand reads float32 x and writes fp16, shrink reads fp16 and writes
 *       float32 y (and the mpjpe of gast_forward_mpjpe).  Each computes in fp32 and rounds once.  Outputs move by
 *       ~2e-3 of max |y| (DESIGN.md §4.1).  The stream rings are fp16 (the input history stays float32), so
 *       gast_stream_state_bytes depends on it and a state must be used at the precision it was sized at;
 *       gast_stream_export / _import convert (snapshots stay float32), which is how streams change precision.
 *       Inference only, like 1.  Setting it fails, before anything is launched, on a half handle (GAST_F16, which
 *       has its own fp16 arithmetic), a sub-module kind, a handle forced onto the FFMA core, channels that are not a
 *       multiple of 32 or more than 20 joints: the half form's own limits.
 * Any other value fails.  Everything else (expand, row-dots, the attention mix, shrink, GEMMs the tensor-core core
 * does not take, every GEMM under gast_set_gemm_core(h, 1)) stays fp32 at 0 and 1.  Like a core switch it needs no
 * gast_prepare and costs nothing; between 0 and 1 it does not invalidate stream `state`. */
enum { GAST_PRECISION_F16 = 16 };
int gast_set_precision(gast_t* h, int32_t mode);

/* Activation type of the model forward (MODEL kind only):
 *   GAST_F32 (default): every activation, x and y are float32.
 *   GAST_F16: gast_forward, gast_forward_chunked, gast_workspace_bytes and gast_chunked_workspace_bytes(.., 0) take
 *       __half x and y, and every activation in the workspace is fp16 (the attention row dots stay fp32).  The
 *       parameters are still bound as float32 and folded exactly as before.  Every GEMM runs the tensor-core core's
 *       half form: one fp16 product per multiply-add on fp16(W 2^s_W) (the fp32-grade form's weight copy), fp32
 *       accumulation, the weight scale and the fused epilogues applied in fp32, each stored value rounded once to fp16
 *       (DESIGN.md §4.1).  Expand, row dots, the attention mix and shrink read and write fp16 and compute in fp32.
 *       A GEMM the tensor-core core does not take (widths that are not multiples of 32) fails the forward: there is no
 *       FFMA core in half.  Inference only: while it is set, gast_forward_mpjpe, gast_forward_train, gast_backward,
 *       gast_backward_input, gast_eval_backward(_chunked), gast_chunked_workspace_bytes(.., 1), the training and
 *       eval-backward workspace queries and every gast_stream_* entry fail, as do gast_set_gemm_core(h, 1) and
 *       gast_set_precision(h, 1) (TF32 and half are separate modes: neither picks the other).  Setting GAST_F16 fails
 *       on a sub-module kind, a TF32 or fp16-precision handle, one forced onto the FFMA core, channels that are not a multiple of 32
 *       (the widths the half form takes) or more than 20 joints (the attention mix then needs the fused epilogue,
 *       which has no half form), before anything is launched.
 * bf16 is not offered (8 significant bits are about a centimetre on these poses).  Needs no gast_prepare. */
enum { GAST_F32 = 0, GAST_F16 = 1 };
int gast_set_activation_dtype(gast_t* h, int32_t dtype);

/* Arithmetic of training and of every gradient: gast_forward_train, gast_backward, gast_backward_input and
 * gast_eval_backward (its recompute of the activations included):
 *   0 = fp32-grade (default): 3xTF32 tensor-core GEMMs, weight gradients in exact fp32 (FFMA).
 *   1 = TF32: every tensor-core GEMM (forward and input-gradient) is one TF32 product per multiply-add, and every
 *       weight gradient whose N and K are multiples of 32 runs on a TF32 tensor-core kernel (wgrad_tc.cuh): operands
 *       rounded to nearest tf32, fp32 accumulation, the same row splits and fixed-order reduction, so results repeat
 *       bit for bit.  Gradients move by ~1e-3 relative (DESIGN.md §4.3).  The other weight gradients (the 8-wide
 *       row-dot one, the expand conv's), BatchNorm statistics, dropout, the SemCH / attention parameter gradients, the
 *       shrink and the expand stay fp32.
 * Under gast_set_gemm_core(h, 1) everything stays fp32 FFMA in either mode.  While it is 0, a handle whose inference
 * precision (gast_set_precision) is 1 refuses training; at 1 training runs whatever the inference precision.  Any
 * other value fails.  Needs no gast_prepare, leaves no state behind and does not touch stream `state`. */
int gast_set_train_precision(gast_t* h, int32_t mode);

/* Number of weight gradients of the last gast_forward_train + gast_backward(_input) pair, or of the last
 * gast_eval_backward, that ran on the TF32 tensor-core weight-gradient kernel; 0 after any other forward-type call
 * (counted like gast_last_launch_count). */
int32_t gast_last_wgrad_tc_launch_count(const gast_t* h);

/* ---- test-time augmentation around the forward (the caller-side steps of reconstruction.evaluate /
 * main.evaluate, kept on the device) -----------------------------------------------------------------
 * gast_tta_prepare: UnchunkedGenerator.next_epoch(augment=True) (common/generators.py:210-233):
 *   seq (T,J,F) -> out (2, T+2*pad, J, F): edge padding (pad+causal_shift left, pad-causal_shift right)
 *   and the mirrored twin (feature 0 negated, kps_left[k] <-> kps_right[k] swapped).
 * gast_tta_merge: main.py:314-318: pred (2,T,J,3) -> out (T,J,3) = mean(pred[0], un-flipped pred[1]).
 * Index lists are host arrays of n_sym entries. */
int gast_tta_prepare(const float* seq, float* out, int32_t T, int32_t J, int32_t F, int32_t pad, int32_t causal_shift,
                     int32_t n_sym, const int32_t* kps_left, const int32_t* kps_right, void* stream);
int gast_tta_merge(const float* pred, float* out, int32_t T, int32_t J, int32_t n_sym, const int32_t* joints_left,
                   const int32_t* joints_right, void* stream);

/* ---- training (SpatioTemporalModelOptimized1f in train() mode, main.py:213-243) -------------------
 * gast_forward_train: forward with batch-statistics BatchNorm (running stats of the bound buffers
 *   are updated in place, momentum 0.1) and Dropout(p) driven by `seed`; keeps what the backward
 *   needs in `workspace` (must stay untouched until gast_backward).  x (B,T,J,F) -> y (B,T_out,J,3).
 * gast_backward: dy (B,T_out,J,3) -> gradient of every parameter, WRITTEN (not accumulated) into the
 *   buffers bound with gast_bind_grads (same keys as gast_bind; buffers/running stats have none).
 * gast_backward_input: the same backward, plus dL/dx (B,T,J,F) into dx when dx is not null.  param_grads = 0
 *   computes no parameter gradient: no weight-gradient kernel runs and no gradient buffer need be bound.
 *   gast_backward(h, dy, ws, n, st) is gast_backward_input(h, dy, NULL, 1, ws, n, st).  The backward is refused
 *   before any launch unless workspace_bytes is at least gast_train_workspace_bytes of its forward's B, T and
 *   dropout_p: the size that forward checked, which bounds every backward of it.
 * A missing or wrong-sized parameter binding, and for a backward with param_grads a missing or wrong-sized gradient
 *   buffer, is refused before any launch, and the error names the key.  A refused gast_forward_train leaves the
 *   running statistics untouched; a refused backward keeps the saved forward, so the caller can fix the binding and
 *   call it again.  gast_train_workspace_bytes needs nothing bound.
 * Both models train on their own schedule (strided for Optimized1f, dilated or dense otherwise; main.py:166-175). */
int gast_bind_grads(gast_t* h, int32_t n, const char* const* keys, void* const* dev_ptrs, const int64_t* numel);
size_t gast_train_workspace_bytes(gast_t* h, int32_t B, int32_t T, float dropout_p);
int gast_forward_train(gast_t* h, const float* x, float* y, int32_t B, int32_t T, float dropout_p, uint64_t seed,
                       void* workspace, size_t workspace_bytes, void* stream);
int gast_backward(gast_t* h, const float* dy, void* workspace, size_t workspace_bytes, void* stream);
int gast_backward_input(gast_t* h, const float* dy, float* dx, int32_t param_grads, void* workspace,
                        size_t workspace_bytes, void* stream);

/* ---- eval-mode gradients (model.eval(): BatchNorm on the running statistics, no dropout) ---------------------
 * gast_eval_backward: backward of gast_forward(h, x, ..., B, T, strided_now) for the output gradient dy
 *   (B,T_out,J,3).  Recomputes what it needs from x with a training-path forward whose BatchNorms use the running
 *   statistics (same schedule as gast_forward: with strided_now a dilated model computes only the positions its
 *   output needs), then writes the parameter gradients (param_grads != 0) into the buffers bound with
 *   gast_bind_grads and dL/dx (B,T,J,F) into dx (may be null).  Running statistics are only read.  The eval
 *   forward itself is unchanged; nothing is kept between it and this call.  Like gast_forward_train it rewrites
 *   the attention constants gast_prepare derives, from the same parameters (so with the same values).
 *   A bad parameter binding, or with param_grads a bad gradient buffer, is refused before any launch.
 * gast_eval_backward_workspace_bytes: scratch for it with parameter gradients (the input-only call needs less); it
 *   needs nothing bound.
 * gast_last_launch_count afterwards: the GEMM and weight-gradient kernels this call enqueued. */
size_t gast_eval_backward_workspace_bytes(gast_t* h, int32_t B, int32_t T, int32_t strided_now);
int gast_eval_backward(gast_t* h, const float* x, const float* dy, float* dx, int32_t param_grads, int32_t B, int32_t T,
                       int32_t strided_now, void* workspace, size_t workspace_bytes, void* stream);

/* ---- the same in bounded memory: long recordings and large batches (MODEL kind) ------------------------------
 * A chunked call covers the (clip, output frame) grid of gast_forward(h, x, ..., B, T, strided_now) in passes of at
 * most max_frames output positions; gast_eval_backward and its workspace query are the case of one pass.  With
 * T_out = gast_out_frames(h, T, strided_now): if T_out <= max_frames a pass covers max_frames / T_out whole clips;
 * otherwise every clip is covered by windows of max_frames output frames (the last may be shorter), and the window
 * of output frames [t0, t0 + K) reads the input frames that map to them, [t0*S, t0*S + (K-1)*S + rf) with
 * rf = gast_receptive_field(h) and S the schedule's output stride (1 dilated or dense, rf strided).  Passes run clip
 * by clip, window by window; every output position falls in exactly one.
 * gast_chunked_workspace_bytes: scratch for gast_forward_chunked (with_backward = 0) or for
 *   gast_eval_backward_chunked with parameter gradients (with_backward != 0; the input-only call needs less); 0 when
 *   the call would be refused.  It needs nothing bound.  For a fixed max_frames it does not depend on T once a clip
 *   needs windows, nor on B once one pass is full (with_backward: once there are two passes, since a single pass is
 *   gast_eval_backward_workspace_bytes).
 * gast_forward_chunked: y (B,T_out,J,3) is bitwise gast_forward's (a GEMM row does not depend on its tile).
 * gast_eval_backward_chunked: the contract of gast_eval_backward.  Each pass is that call's frozen-BatchNorm
 *   recompute and backward on its slice of x and dy.  Parameter gradients are WRITTEN into the buffers bound with
 *   gast_bind_grads: the first pass writes them, every later pass writes into the workspace and one multi-tensor
 *   kernel adds them, in pass order.  dx (may be null) is written: a clip's windows overlap by rf - 1 input frames,
 *   so with windows dx is zeroed first and every window adds its own.  Handle kind, max_frames >= 1, B, T, the
 *   parameter and gradient bindings and the workspace size are checked before the first launch; a refused call
 *   changes no buffer.  With a single pass (max_frames >= B * T_out) it is gast_eval_backward: the same workspace
 *   size, kernels and order; with several passes the results differ from it by summation order only.  Both repeat
 *   bit for bit where gast_eval_backward does: on the strided schedule.  On the dilated and dense schedules the taps
 *   of a temporal conv overlap and their adjoints are added with float atomics, so there either call varies in the
 *   last bits from run to run. */
size_t gast_chunked_workspace_bytes(gast_t* h, int32_t B, int32_t T, int32_t strided_now, int32_t max_frames,
                                    int32_t with_backward);
int gast_forward_chunked(gast_t* h, const float* x, float* y, int32_t B, int32_t T, int32_t strided_now,
                         int32_t max_frames, void* workspace, size_t workspace_bytes, void* stream);
int gast_eval_backward_chunked(gast_t* h, const float* x, const float* dy, float* dx, int32_t param_grads, int32_t B,
                               int32_t T, int32_t strided_now, int32_t max_frames, void* workspace,
                               size_t workspace_bytes, void* stream);
/* Optional device-side dropout state: one uint64 on the device (caller-owned, may be null to unset) that is added to
 * `seed` by every dropout kernel and advanced once per gast_forward_train.  With it a CUDA graph that captured a
 * training step (frozen kernel arguments) draws a fresh mask at every replay. */
int gast_set_dropout_state(gast_t* h, void* dev_u64);

/* ---- real-time streams (SURVEY.md 8f N4; gen_skes.py:43-69, tools/inference.py:19-110) -------------------
 * The reference's real-time model is a causal SpatioTemporalModelOptimized1f re-run on the last
 * receptive_field frames for every new frame.  Here a pushed frame costs ONE new position per layer: `state`
 * (caller-owned device memory, gast_stream_state_bytes, contents irrelevant before the first push) holds per
 * temporal stage a ring of that stage's past inputs for n_streams concurrent streams.  State and workspace
 * sizes are the same for causal and non-causal handles of one architecture.
 * gast_stream_push: x (n_streams, J, in_features) = the newest frame of every stream -> y (n_streams, J, 3) =
 *   its 3D pose, identical to the whole-sequence causal forward on the sequence so far, left-padded by
 *   replicating the stream's first frame (UnchunkedGenerator(pad, causal_shift=pad), common/generators.py:210-221).
 *   step = number of frames pushed into `state` before this one (0, 1, 2, ...; the caller counts).
 *   fresh (n_streams) int32 on the device, or null: non-zero = this frame starts a new sequence on that stream
 *   (must be non-zero for every stream at step 0).  MODEL handles with causal = 1 only; all work on `stream`.
 *   The rings hold layer inputs computed with the weights of the pushes that wrote them.  A gast_prepare (after
 *   new weights or BatchNorm statistics were bound) therefore invalidates `state`: unless the next push marks
 *   every stream fresh, it mixes old and new weights for up to receptive_field - 1 pushes.  Nothing checks this
 *   here; gast_b200.realtime.CausalStream refuses such a push.  gast_set_gemm_core and gast_set_precision between 0
 *   and 1 do not invalidate `state`.  At the fp16 precision the rings are fp16 and the state is smaller: a state
 *   sized at one ring type must not be pushed at the other (gast_stream_export / _import move streams across). */
size_t gast_stream_state_bytes(gast_t* h, int32_t n_streams);
size_t gast_stream_workspace_bytes(gast_t* h, int32_t n_streams);
int gast_stream_push(gast_t* h, void* state, int64_t step, const float* x, float* y, int32_t n_streams,
                     const int32_t* fresh, void* workspace, size_t workspace_bytes, void* stream);
/* gast_stream_push_ex: gast_stream_push for causal AND non-causal MODEL handles (not dense), with a hold mask.
 *   y[s] is the pose of the frame pushed gast_stream_latency(h) pushes earlier on stream s: 0 for a causal
 *   model, pad = (receptive_field - 1) / 2 for a non-causal one.  A sequence's poses equal the reference's
 *   UnchunkedGenerator([seq], pad, causal_shift = causal ? pad : 0) + model forward when the caller
 *     - marks the sequence's first frame fresh (left padding: copies of the first frame), and
 *     - after its last frame makes `latency` more pushes with hold[s] != 0 (right padding: copies of the last
 *       frame).  Those pushes return the sequence's last `latency` poses.
 *   The first `latency` outputs after a fresh frame belong to frames before the sequence and are meaningless.
 *   hold (n_streams) int32 on the device, or null: non-zero = stream s re-appends its own newest frame and
 *   ignores x[s]; fresh wins over hold.  gast_stream_push(...) is gast_stream_push_ex(..., hold = NULL, ...)
 *   after refusing non-causal handles.  Same step / fresh / weight-change rules as gast_stream_push.
 *   Test-time augmentation (tools/inference.py:19-110: augment=True, un-flip and average) composes from the TTA
 *   entries with T = n_streams: gast_tta_prepare(x, x2, n, J, F, pad = 0, shift = 0, kps lists) writes
 *   x2 (2, n, J, F) = [original | mirrored]; push x2 as 2n streams into a state sized for 2n streams, with the
 *   fresh and hold masks repeated for both halves; gast_tta_merge(y2, y, n, J, joints lists) averages
 *   y2 (2n, J, 3) into y (n, J, 3).
 * gast_stream_latency: 0 (causal), (receptive_field - 1) / 2 (non-causal), -1 for a handle that cannot stream. */
int32_t gast_stream_latency(const gast_t* h);
int gast_stream_push_ex(gast_t* h, void* state, int64_t step, const float* x, float* y, int32_t n_streams,
                        const int32_t* fresh, const int32_t* hold, void* workspace, size_t workspace_bytes,
                        void* stream);
/* gast_stream_push_chunk: K frames per stream in one call.  x (n_streams, K, J, in_features) -> y (n_streams, K, J, 3),
 *   equal up to float rounding to K calls of gast_stream_push_ex at steps step, step+1, ..., step+K-1 with x[:, k],
 *   fresh at k = 0 only and hold[:, k]; it also leaves `state` as those K pushes would.  So single pushes and chunks
 *   can be mixed freely on one state, and step advances by K.  Same state (gast_stream_state_bytes), handles (causal
 *   or not, not dense) and step / fresh / weight-change rules as gast_stream_push_ex.  The launch count does not
 *   depend on n_streams or K: the work is one forward over n_streams*K positions, so frames that are already
 *   available (a burst, catching up, a recorded sequence) cost far less than K single pushes.
 *   fresh (n_streams) int32 or null: applies to frame 0 of the chunk (start sequences only at chunk boundaries).
 *   hold (n_streams, K) int32 or null: hold[s, k] != 0 = frame k of stream s repeats that stream's newest frame
 *   (which may be a held frame earlier in the chunk) and x[s, k] is not read; fresh wins over hold at k = 0.
 *   K >= 1 and n_streams*K*J < 2^31.  The workspace is gast_stream_chunk_workspace_bytes(h, n_streams, K) bytes
 *   (0 for invalid arguments; it grows with K, so a workspace sized for K serves every smaller K).
 *   With test-time augmentation: gast_tta_prepare / gast_tta_merge with T = n_streams*K: the (2, n*K, J, F) layout is
 *   2n streams of K frames, with the masks repeated for both halves. */
size_t gast_stream_chunk_workspace_bytes(gast_t* h, int32_t n_streams, int32_t K);
int gast_stream_push_chunk(gast_t* h, void* state, int64_t step, const float* x, float* y, int32_t n_streams,
                           int32_t K, const int32_t* fresh, const int32_t* hold, void* workspace,
                           size_t workspace_bytes, void* stream);
/* gast_stream_peek: provisional poses of the frames a non-causal stream has not returned yet, without pushing.
 *   y (n_streams, K, J, 3) is what K calls of gast_stream_push_ex at steps step, step+1, ..., step+K-1 would return
 *   with fresh = NULL and hold[s] = 1 for every stream; `state` is not modified (byte for byte), and step does not
 *   advance.  So, for a stream that pushed frames 0 .. l-1 of its current sequence, row k is the pose of frame
 *   l - latency + k as the reference computes it for the sequence cut at frame l - 1 (UnchunkedGenerator's right
 *   padding by copies of the newest frame).  The final poses still come from the pushes, latency pushes later.
 *   Lookahead: for poses L frames behind the newest (0 <= L < latency) peek K = latency - L and take row K-1; with
 *   K = latency the last row is the newest frame.
 *   1 <= K <= gast_stream_latency(h) (so a causal handle, whose latency is 0, is refused) and step >= 1.  Same
 *   handles, state and weight-change rule as gast_stream_push_chunk; the workspace is
 *   gast_stream_chunk_workspace_bytes(h, n_streams, K) bytes.  The cost is that of a chunk of K frames; the launch
 *   count does not depend on n_streams or K.
 *   Test-time augmentation: peek the 2n-stream state (no gast_tta_prepare: a peek has no new input), then
 *   gast_tta_merge(y2, y, n * K, J, ...) with y2 (2, n, K, J, 3). */
int gast_stream_peek(gast_t* h, const void* state, int64_t step, float* y, int32_t n_streams, int32_t K,
                     void* workspace, size_t workspace_bytes, void* stream);
/* gast_stream_push_subset / gast_stream_peek_subset: any subset of the streams, each at its own frame count.
 *   The lockstep entries above advance every stream of `state` by the same frames.  These take m distinct streams
 *   streams[0..m) (host array, indices into [0, n_streams)) with their own counts steps[0..m) (host array: the frames
 *   pushed into that stream so far; the caller keeps the counts, as it keeps `step` for the lockstep entries).
 *   Row i of x (m, K, J, in_features), y (m, K, J, 3), fresh (m) and hold (m, K) (device, null as for
 *   gast_stream_push_chunk) belongs to stream streams[i].  A subset push returns, and leaves stream streams[i]'s part
 *   of `state` as, what gast_stream_push_chunk returns and leaves on a state holding that stream alone at step
 *   steps[i].  Every byte of an unlisted stream (its input history and every ring slot of its rows) is unchanged.
 *   A stream whose own count is 0 must be fresh.  gast_stream_peek_subset is gast_stream_peek for the listed streams
 *   on the same terms: 1 <= K <= gast_stream_latency(h), steps[i] >= 1, nothing written to `state`.
 *   Refused (gast_last_error) before any launch: m outside [1, n_streams], a stream outside [0, n_streams) or listed
 *   twice, a negative step (peek: a step below 1).  The work is one chunk forward over m*K positions, so it costs
 *   what the listed streams cost, not what n_streams cost; the launch count depends on neither n_streams, m nor K.
 *   The workspace is gast_stream_subset_workspace_bytes(h, m, K) bytes (it grows with m and K; 0 for bad arguments),
 *   independent of n_streams.  Listing every stream in order at one step runs exactly gast_stream_push_chunk's (or
 *   gast_stream_peek's) kernels on the same rows.
 *   Mixing with the lockstep entries: gast_stream_push(_ex), _push_chunk and _peek remain valid on the same state
 *   only while every stream's own count equals their `step`; after counts diverge, use the subset entries.
 *   Test-time augmentation: list 2m library streams [streams, streams + n] of the 2n-stream state with the steps
 *   repeated for both halves, gast_tta_prepare / gast_tta_merge with T = m*K, masks repeated for both halves. */
size_t gast_stream_subset_workspace_bytes(gast_t* h, int32_t m, int32_t K);
int gast_stream_push_subset(gast_t* h, void* state, int32_t n_streams, const int32_t* streams, const int64_t* steps,
                            int32_t m, int32_t K, const float* x, float* y, const int32_t* fresh, const int32_t* hold,
                            void* workspace, size_t workspace_bytes, void* stream);
int gast_stream_peek_subset(gast_t* h, const void* state, int32_t n_streams, const int32_t* streams,
                            const int64_t* steps, int32_t m, int32_t K, float* y, void* workspace,
                            size_t workspace_bytes, void* stream);
/* gast_stream_push_device / gast_stream_peek_device: the subset entries with the frame counts kept on the device, so
 *   that a CUDA graph can capture a tick and replay it at every later count.
 *   counts (n_streams) int64 on the device: what `steps` is for the subset entries, the frames pushed into each stream
 *   so far (held frames included).  active (n_streams) int32 on the device, or null (every stream active).  x
 *   (n_streams, K, J, in_features), y (n_streams, K, J, 3), fresh (n_streams) and hold (n_streams, K) are on the
 *   device, indexed by stream, null masks as for gast_stream_push_chunk.
 *   A push returns in the rows of the active streams, and leaves in their bytes of `state`, exactly what
 *   gast_stream_push_subset returns and leaves when it lists the active streams in ascending order at steps counts[s]
 *   (bit for bit), and adds K to counts[s] of every active stream on the device.  An inactive stream's row of x is not
 *   read, its bytes of `state` and its count are unchanged, and its rows of y are unspecified.  A peek returns what
 *   gast_stream_peek_subset returns for the active streams with counts[s] >= 1 (1 <= K <= gast_stream_latency(h), so
 *   not for a causal handle) and writes nothing to `state` or `counts`.
 *   Device values cannot make a kernel address memory outside `state`, the workspace or the operands: a count of 0
 *   makes its stream fresh (its ring is never read), a negative count is taken as 0 (a push then leaves it at K), and
 *   counts up to 2^62 work.  The calls read no device data on the host, allocate nothing, do not synchronise and copy
 *   nothing from host memory; every refusal (null handle, state, counts, x or y, n_streams < 1, K < 1, a peek's K
 *   outside [1, latency], a dense, non-MODEL or unprepared handle, a workspace smaller than
 *   gast_stream_device_workspace_bytes(h, n_streams, K)) comes before the first launch.  So a call made during stream
 *   capture either fails at capture time or records a graph that is right at every replay, provided the handle sees
 *   no gast_bind / gast_prepare in between (new weights: capture again) and gast_set_timing is off while capturing.
 *   The launch count is that of the chunk or peek call plus one, whatever n_streams, K and the active set.
 *   These entries mix freely with the subset entries on one state, as long as the host's steps equal the device
 *   counts.  Test-time augmentation: 2n_streams library streams with counts, active and the masks repeated for both
 *   halves, as for the subset entries. */
size_t gast_stream_device_workspace_bytes(gast_t* h, int32_t n_streams, int32_t K);
int gast_stream_push_device(gast_t* h, void* state, int32_t n_streams, int64_t* counts, const int32_t* active,
                            int32_t K, const float* x, float* y, const int32_t* fresh, const int32_t* hold,
                            void* workspace, size_t workspace_bytes, void* stream);
int gast_stream_peek_device(gast_t* h, const void* state, int32_t n_streams, const int64_t* counts,
                            const int32_t* active, int32_t K, float* y, void* workspace, size_t workspace_bytes,
                            void* stream);
/* gast_stream_export / gast_stream_import: move streams between states with their history, e.g. into a state of
 *   another n_streams, or between a state driven by the host counts and one driven by device counts.
 *   A stream's SNAPSHOT is its history in time order, gast_stream_snapshot_floats(h) floats:
 *     [input history (k0, J, in_features), oldest first][ring_1 (R_1, J, C_1), oldest first] ... [ring_{L-1}]
 *   with k0 = filter_widths[0], C_i = channels << i, R_i = filter_widths[i] * (filter_widths[0] * ... *
 *   filter_widths[i-1]).  Row j of ring i of a stream whose count is c is its slot (c - R_i + j) mod R_i, so a
 *   snapshot does not depend on the ring phase.  Snapshots are float32 at every precision: an export from fp16 rings
 *   (gast_set_precision(h, 16)) widens them exactly, an import into fp16 rings rounds to nearest, so streams move
 *   between states of either precision.
 *   gast_stream_export writes out (m, snapshot_floats) (device) = the snapshots of streams streams[0..m) at their
 *   counts counts[0..m); `state` is only read.  gast_stream_import writes snapshot in[i] to stream streams[i] at the
 *   target count counts[i] (so it may land at any phase, e.g. at the target state's lockstep step) and writes no
 *   byte of an unlisted stream.  A stream imported at count c' then continues exactly as the exported stream did at
 *   count c, the same for every later push, peek and subset call at counts c' + k (the chunk path reads the rings in
 *   time order; a single-frame lockstep push is bitwise the same when c' = c mod R_max, and equal up to float rounding
 *   otherwise, as the tap-rotated weights differ).  Both need a handle of the architecture that wrote the state
 *   (gast_stream_state_bytes sizes) and no gast_prepare; the history stays that of the weights of the pushes that
 *   wrote it (gast_stream_push's weight-change rule).
 *   streams and counts are host arrays, checked as for gast_stream_push_subset: m in [1, n_streams], streams
 *   distinct and in [0, n_streams), counts >= 1.  Every refusal comes before the first launch.  The workspace is
 *   gast_stream_move_workspace_bytes(h, m) bytes (0 for bad arguments).  Each call is one table copy and one kernel
 *   launch, whatever n_streams, m and the depth of the model.
 *   Test-time augmentation: a stream is two library streams, s and s + n_streams of the 2n-stream state. */
size_t gast_stream_snapshot_floats(gast_t* h);
size_t gast_stream_move_workspace_bytes(gast_t* h, int32_t m);
int gast_stream_export(gast_t* h, const void* state, int32_t n_streams, const int32_t* streams, const int64_t* counts,
                       int32_t m, float* out, void* workspace, size_t workspace_bytes, void* stream);
int gast_stream_import(gast_t* h, void* state, int32_t n_streams, const int32_t* streams, const int64_t* counts,
                       int32_t m, const float* in, void* workspace, size_t workspace_bytes, void* stream);

/* ---- either side of the forward, on the device (SURVEY.md 8f N1-N3) --------------------------------
 * All pointers are device pointers unless marked (host).  Work is enqueued on `stream`.
 *
 * gast_chunk_gather: one training batch of ChunkedGenerator.next_epoch (common/generators.py:93-154).
 *   poses_2d (total_frames,J2,F2) / poses_3d (total_frames,J3,3) = every sequence concatenated along
 *   time; seq_start[n_seq+1] = first frame of each sequence; cameras (n_seq,ncam); pairs (B,4) int32 =
 *   the reference's (seq_i, start_3d, end_3d, flip) tuples.  Writes batch_2d (B,chunk+2*pad,J2,F2)
 *   with edge padding and the horizontal flip (:107-121), batch_3d (B,chunk,J3,3) (:123-135, may be
 *   null) and batch_cam (B,ncam) (:137-144, may be null).  kps_/joints_ lists: (host). */
int gast_chunk_gather(const float* poses_2d, const float* poses_3d, const float* cameras, const int64_t* seq_start,
                      int32_t n_seq, const int32_t* pairs, int32_t B, int32_t chunk, int32_t pad, int32_t causal_shift,
                      int32_t J2, int32_t F2, int32_t J3, int32_t ncam, int32_t n_sym2, const int32_t* kps_left,
                      const int32_t* kps_right, int32_t n_sym3, const int32_t* joints_left, const int32_t* joints_right,
                      float* batch_2d, float* batch_3d, float* batch_cam, void* stream);

/* tools/mpii_coco_h36m.py: mode 0 = coco_h36m (T,17,2)->(T,17,2) (:20-48), 1 = mpii_h36m (T,16,2)->(T,17,2)
 * (:51-59), 2 = coco_h36m_toe_format (T,J_in>=22,2)->(T,19,2) (:62-78), 3 = HumanEva's COCO -> 15 joints
 * (T,17,2)->(T,15,2) (main.py:80-95).  valid (T) int32, may be null:
 * 1 where the frame's coordinate sum is non-zero (the mask the reference takes np.where of). */
int gast_keypoints_convert(const float* kpts, float* out, int32_t* valid, int32_t T, int32_t J_in, int32_t mode,
                           void* stream);

/* The video demo's keypoint repair and placement of the lifted persons (tools/preprocess.py), float32 in the
 * reference's order of operations: bit-identical to it for float32 input.  Minima are taken in two deterministic
 * passes (per-block partials, then a fixed-order finish), so results repeat bit for bit.
 *
 * gast_h36m_coco_format (preprocess.py:47-75): kpts (P,T,17,2) COCO keypoints and scores (P,T,17) of P person slots ->
 *   out_kpts (P,T,17,2) H36M keypoints and valid (P,T) as gast_keypoints_convert mode 0 (:61), out_scores (P,T,17) the
 *   H36M scores (:65-69), keep (P) = 1 where the slot holds a person.  The reference keeps a slot when np.sum(kpts) != 0
 *   (:60); here when some coordinate is non-zero.  The two differ only when non-zero coordinates cancel to exactly 0,
 *   which needs negative pixel coordinates.  The caller drops the slots with keep = 0. */
int gast_h36m_coco_format(const float* kpts, const float* scores, int32_t P, int32_t T, float* out_kpts, float* out_scores,
                          int32_t* valid, int32_t* keep, void* stream);

/* gast_revise_kpts (preprocess.py:78-112): kpts (P,T,J,2), scores (P,T,J), valid (P,T) int32 mask of each person's
 *   valid frames -> out (P,T,J,2): zero outside the valid frames; at a valid frame the pose with the low-confidence
 *   joints among [2, 3, 5, 6] (score < float32(0.3)) replaced as :96-107 do. */
int gast_revise_kpts(const float* kpts, const float* scores, const int32_t* valid, int32_t P, int32_t T, int32_t J,
                     float* out, void* stream);

/* gast_revise_skes (preprocess.py:123-155): pred (sum F_p, J, 3) = every person's prediction packed, person p at rows
 *   offsets[p] .. offsets[p+1]-1 (offsets (host), P+1 entries, offsets[0] = 0); frames (sum F_p) int64 = the frame of
 *   each row (the reference's valid_frames, concatenated); kpts (P,T,J,D) the repaired 2D keypoints (D >= 2, J >= 15)
 *   -> out (P,T,J,3): zero, each row scattered to its frame, moved in x/y by the joint [1,4,11,14] mean displacement
 *   from the person's first frame / 500 (:130-133); with P = 2 both persons moved apart by half their mean distance at
 *   the first frame of person 0 that person 1 also has (:138-147); then z -= min z over the whole output (:153), zero
 *   rows of missing frames included (so the minimum is <= 0 as soon as a person misses a frame, as in the reference).
 *   The first and common frames are found on the device.  Two persons without a common frame, where the reference
 *   raises ValueError, get NaN x and y.  workspace: gast_revise_skes_workspace_bytes(P, T) bytes. */
size_t gast_revise_skes_workspace_bytes(int32_t P, int32_t T);
int gast_revise_skes(const float* pred, const int64_t* frames, const int64_t* offsets, int32_t P, int32_t T, int32_t J,
                     int32_t D, const float* kpts, float* out, void* workspace, size_t workspace_bytes, void* stream);

/* gast_revise_skes_real_time (preprocess.py:158-172): pred (M,17,3) and kpts (M,17,D) of one tick -> out (M,17,3):
 *   x -= (m_x - 3 width/5) / r, y += (m_y - width/5) / r with m the joint [1,4,11,14] mean of the person's keypoints and
 *   r = 500 width/1920, then z -= min z over all M persons.  The constants are computed in double and rounded to
 *   float32, every other step is float32 (NumPy 2 promotion of the reference's Python-float constants).  J != 17 fails,
 *   as the reference hard-codes 17 joints.  workspace: gast_revise_skes_real_time_workspace_bytes(M) bytes. */
size_t gast_revise_skes_real_time_workspace_bytes(int32_t M);
int gast_revise_skes_real_time(const float* pred, const float* kpts, int32_t M, int32_t J, int32_t D, double width, float* out,
                               void* workspace, size_t workspace_bytes, void* stream);

/* common/camera.py:8-19: normalize_screen_coordinates (inverse = 0) / image_coordinates (inverse = 1) on
 * n_points (x,y) pairs. */
int gast_normalize_screen(const float* x, float* out, int64_t n_points, float w, float h, int32_t inverse, void* stream);

/* common/camera.py:27-28 camera_to_world with one rotation for all points: qort(q, x) + t
 * (common/quaternion.py:4-18).  q[4], t[3] (host; t may be null = 0). */
int gast_camera_to_world(const float* x, float* out, int64_t n_points, const float* q, const float* t, void* stream);

/* Dataset preparation (main.py:24-104 load_data, data/prepare_data_h36m.py:113-121) as segmented launches, bit-identical
 * to the reference for float32 input.  Output segment s (s < S) holds rows dst_start[s] .. dst_start[s+1]-1, taken from
 * source rows src_start[s] ..; dst_start (S+1, ascending from 0) and src_start (S) are int64 device arrays, as are the
 * per-segment parameter tables.  An output row whose source row lies outside the input is left unwritten.
 *
 * gast_world_to_camera: world_to_camera (camera.py:22-24) of frames of J points x (n_src_frames,J,3) -> out
 *   (n_out_frames,J,3); qt (S,7) float = {orientation[4], translation[3]} per segment.  root_relative subtracts each
 *   frame's joint 0 from its joints 1.. (main.py:33).  torch's CPU cross product rounds each component as
 *   fma(a1, b2, -(a2*b1)); the kernel does the same.
 * gast_project_to_2d: project_to_2d (camera.py:31-62) of n_points camera-space points x (n,3) -> out (n,2); here the
 *   segments count points (seg_start, S+1) and intrinsics (S,9) = {f[2], c[2], k[3], p[2]} per segment.
 * gast_project_to_2d_backward: grad_x (n,3) = dL/dx given grad_out (n,2) = dL/dout, evaluated in double.
 * gast_normalize_screen_segments: normalize_screen_coordinates (camera.py:8-12) of frames of P points of F >= 2 floats,
 *   x (n_src_frames,P,F) -> out (n_out_frames,P,F): channels 0 and 1 with wh (S,2) double = {w, h/w} per segment,
 *   the others copied.  from_image = 1 takes each point through image_coordinates (camera.py:15-19) and float32
 *   first: the ground-truth keypoints' round trip. */
int gast_world_to_camera(const float* x, int64_t n_src_frames, int32_t J, const int64_t* src_start,
                         const int64_t* dst_start, const float* qt, int32_t S, int64_t n_out_frames, int32_t root_relative,
                         float* out, void* stream);
int gast_project_to_2d(const float* x, int64_t n_points, const int64_t* seg_start, const float* intrinsics, int32_t S,
                       float* out, void* stream);
int gast_project_to_2d_backward(const float* x, int64_t n_points, const int64_t* seg_start, const float* intrinsics,
                                int32_t S, const float* grad_out, float* grad_x, void* stream);
int gast_normalize_screen_segments(const float* x, int64_t n_src_frames, int32_t P, int32_t F, const int64_t* src_start,
                                   const int64_t* dst_start, const double* wh, int32_t S, int64_t n_out_frames,
                                   int32_t from_image, float* out, void* stream);

/* common/loss.py:5-11 mpjpe: *loss = mean_i ||pred_i - target_i|| over n_points rows of D (<= 4) coordinates;
 * when dpred is not null it receives grad_scale * d loss / d pred (the backward of the same pass).
 * workspace: gast_mpjpe_workspace_bytes() bytes of scratch. */
size_t gast_mpjpe_workspace_bytes(void);
int gast_mpjpe(const float* pred, const float* target, int64_t n_points, int32_t D, float* loss, float* dpred,
               float grad_scale, void* workspace, void* stream);

/* common/loss.py:14-53 p_mpjpe: per_frame[n] = mean joint distance of frame n after the similarity
 * (Procrustes) alignment of pred[n] (J,3) to target[n]; the reference's scalar is the mean of per_frame. */
int gast_p_mpjpe(const float* pred, const float* target, int32_t N, int32_t J, float* per_frame, void* stream);

/* Scores of a test set, per segment (main.py:299-353 evaluate; common/loss.py:56-90 euclidean_losses, pck, auc).
 * pred, target (N,J,3) float32 on the device, 1 <= J <= 32 (>= 3 with procrustes).  seg_start (S+1) host int64:
 * 0 = seg_start[0] <= ... <= seg_start[S] = N; segment s is frames seg_start[s] .. seg_start[s+1]-1.  thresholds:
 * n_thr (<= 64) host float32, none NaN.  rows (S, 3+J+n_thr) float64 on the device receives per segment
 *   [frames, sum_f mpjpe_f, sum_f p_mpjpe_f, sum_f dist_fj for j < J, count(dist_fj < thresholds[k]) for k < n_thr]
 * with dist = sqrt((dx*dx + dy*dy) + dz*dz) in float32, every step rounded (torch's CPU order), mpjpe_f the mean of a
 * frame's dist in double, and p_mpjpe_f gast_p_mpjpe's value of the frame (0 with procrustes = 0).  zero_root reads
 * target joint 0 as 0 (main.py:327) without writing it.  dist (N,J) float32 on the device, or null, receives every
 * dist.  The sums run in float64 in a fixed order: a segment's row depends only on its own frames, so it is the same
 * bits whatever other segments the call holds.  workspace: gast_pose_metrics_workspace_bytes(S, J, n_thr, N) bytes
 * on the device.  Every argument is checked on the host before the first launch. */
size_t gast_pose_metrics_workspace_bytes(int32_t S, int32_t J, int32_t n_thr, int64_t N);
int gast_pose_metrics(const float* pred, const float* target, int64_t N, int32_t J, const int64_t* seg_start, int32_t S,
                      const float* thresholds, int32_t n_thr, int32_t zero_root, int32_t procrustes, double* rows,
                      float* dist, void* workspace, size_t workspace_bytes, void* stream);

/* Animation frames of the reconstruction (tools/vis_h36m.py:58-249 and tools/visualization.py:84-227
 * render_animation), rasterised.  Frame f < F of out (F, S, S*(1+P), 3) uint8 on the device is source frame f0+f:
 * the input panel (S x S) and then P = (flags & GAST_RENDER_SHARED_PANEL ? 1 : n_pose) 3D panels.
 *   keypoints (n_kp_frames, M, J, 2) float32 in image pixels; poses (n_pose, n_pose_frames, J, 3) float32 world
 *   coordinates; video (n_video_frames, Hin, Win, 3) uint8 or null (a black Hin x Win image); all on the device.
 *   parents (J), colors (J, 3) RGB of the bone ending at each joint, right (n_right): host arrays.  J <= 32,
 *   M*J <= 256, n_pose <= 8 (shared: n_pose*J <= 256).  Bones j = 1 .. n_bones-1 with parents[j] >= 0 are drawn.
 *   flags: GAST_RENDER_SHARED_PANEL draws every pose in one panel with x, y limits +-radius (else +-radius/2; z in
 *   [0, radius]); GAST_RENDER_FOLLOW_ROOT centres each panel's x, y limits on its pose's joint 0 at every frame
 *   (visualization.py:166-167); GAST_RENDER_BONES_2D draws the 2D bones (pink) under the joint discs.
 *   View: elevation elev and azimuth azim in degrees, eye distance dist in units of the axis box (ax.dist).
 * Each pixel is written by one thread, with no atomics: the bytes repeat from call to call, and a frame's bytes do not
 * depend on f0 and F.  Formulas in DESIGN.md §8.5.
 * gast_render_geometry: the call's geometry as float32 geo[20] on the host: [0..11] the 3D panels' rows
 *   (sx, sy, dz) = M (x, y, z, 1), [12..14] the input image's scale and offsets (ox, oy), [15..18] the coverage
 *   edges of the 3D bones, the 2D bones, the disc fill and the disc edge, [19] S/2.
 * gast_downsample_frames: downsample_tensor (vis_h36m.py:53-55) of x (n_in_frames, frame_elems) -> out
 *   (n_in_frames / factor, frame_elems) on the device; dtype 0 = float32 (numpy's float32 mean), 1 = uint8 (numpy's
 *   mean then astype('uint8')). */
#define GAST_RENDER_SHARED_PANEL 1
#define GAST_RENDER_FOLLOW_ROOT 2
#define GAST_RENDER_BONES_2D 4
int gast_render_geometry(int32_t S, float dpi, int32_t Hin, int32_t Win, float elev, float azim, float radius,
                         float dist, int32_t shared, float* geo);
int gast_render_frames(const float* keypoints, int64_t n_kp_frames, int32_t M, int32_t J, const float* poses,
                       int32_t n_pose, int64_t n_pose_frames, const uint8_t* video, int64_t n_video_frames, int32_t Hin,
                       int32_t Win, const int32_t* parents, const uint8_t* colors, const int32_t* right, int32_t n_right,
                       int32_t n_bones, int32_t S, float dpi, float elev, float azim, float radius, float dist,
                       int32_t flags, int64_t f0, int32_t F, uint8_t* out, void* stream);
int gast_downsample_frames(const void* x, int64_t n_in_frames, int64_t frame_elems, int32_t factor, int32_t dtype,
                           void* out, void* stream);

/* The 2D pose net's input crops and its heatmap decode (lib/pose/hrnet/pose_estimation/gen_kpts.py:234-256).
 * gast_person_crops: PreProcess (lib/pose/hrnet/lib/utils/utilitys.py:140-170) of n boxes.  Record r crops frame
 *   frame_index[r] of frames (n_frames, H, W, 3) uint8 (BGR as cv2 reads it; RGB with GAST_CROP_RGB_INPUT) by the
 *   forward 2x3 matrix forward_mats[6r..6r+5] (what cv2.warpAffine receives) into out (n, 3, out_h, out_w) float32:
 *   cv2.warpAffine(frame, M, (out_w, out_h), flags=INTER_LINEAR) with a constant 0 border, ToTensor and
 *   Normalize(mean=[0.485, 0.456, 0.406], std=[0.229, 0.224, 0.225]) bit for bit, the statistics applied to the BGR
 *   planes in order.  Planes in the frame's BGR order, or with GAST_CROP_NET_ORDER in the order the net receives
 *   (inputs[:, [2, 1, 0]]).  A frame index outside [0, n_frames) crops a black frame.  Frame and crop sides <= 32767.
 * gast_heatmap_decode: get_final_preds (lib/pose/hrnet/lib/utils/inference.py:21-82) of heatmaps (n, J, hh, hw)
 *   float32 with the inverse (heatmap -> frame) 2x3 matrices inverse_mats (n, 6) double: preds (n, J, 2) and maxvals
 *   (n, J, 1) float32, bit for bit; post_process 1 = TEST.POST_PROCESS (the quarter-pixel shift).  J <= 32, sides <=
 *   256.
 * Device pointers, the caller's stream, no allocation or synchronisation; calls repeat bit for bit and a record's
 * result does not depend on the others.  Formulas in DESIGN.md §8.6. */
#define GAST_CROP_RGB_INPUT 1
#define GAST_CROP_NET_ORDER 2
int gast_person_crops(const uint8_t* frames, int64_t n_frames, int32_t H, int32_t W, const int32_t* frame_index,
                      const double* forward_mats, int32_t n, int32_t out_w, int32_t out_h, int32_t flags, float* out,
                      void* stream);
int gast_heatmap_decode(const float* heatmaps, const double* inverse_mats, int32_t n, int32_t J, int32_t hh,
                        int32_t hw, int32_t post_process, float* preds, float* maxvals, void* stream);

/* The person detector's input and output handling (lib/detector/yolov3/human_detector.py:106-157).
 * gast_letterbox: preprocess.prep_image (lib/detector/yolov3/preprocess.py:9-38) of n frames (n, H, W, 3) uint8 (BGR
 *   as cv2 reads them; RGB with GAST_LETTERBOX_RGB_INPUT) into out (n, 3, D, D) float32 RGB planes: cv2.resize(
 *   INTER_CUBIC) to new_w x new_h (OpenCV's own path, not IPP's), pasted at ((D - new_w) / 2, (D - new_h) / 2) into a
 *   canvas of 128, each value u8 / 255 correctly rounded.  new_w = int(W * min(D / W, D / H)) as the reference's double
 *   expression gives it, new_h likewise, 1 .. D.  Sides <= 32767; D a multiple of 32 above 32.
 * gast_person_detections: write_results(pred, confidence, 80, nms=True, nms_conf=nms_thresh, det_hm=True)
 *   (lib/detector/yolov3/util.py:107-225) of each frame's predictions (n, N, 85) float32 (Darknet.forward's output),
 *   N = 3 * sum((D / s)^2, s = 32, 16, 8), then yolo_human_det's rescale to frame_sizes (n, 2) int32 (W, H), clamp to
 *   the frame and round(v, 2): boxes (n, max_det, 4), scores (n, max_det) (the objectness) in the reference's order,
 *   zero past the count; counts (n) the number of survivors, which may exceed max_det.  GAST_DETECT_RAW leaves the
 *   boxes as write_results' corners in the D x D input.  Optional: max_conf (n, max_det) write_results' class score
 *   column; persons (n) the rows that reach its person filter (its early return when 0).  Objectness ties keep the
 *   lower prediction index first.  N * 9 bytes of shared memory (D <= 640).
 * Device pointers, the caller's stream, no allocation or synchronisation; calls repeat bit for bit and a frame's
 * result does not depend on the others.  Formulas in DESIGN.md §8.7. */
#define GAST_LETTERBOX_RGB_INPUT 1
#define GAST_DETECT_RAW 1
int gast_letterbox(const uint8_t* frames, int32_t n, int32_t H, int32_t W, int32_t D, int32_t new_w, int32_t new_h,
                   int32_t flags, float* out, void* stream);
int gast_person_detections(const float* predictions, int32_t n, int32_t N, int32_t attrs, int32_t D,
                           const int32_t* frame_sizes, float confidence, float nms_thresh, int32_t max_det,
                           int32_t flags, float* boxes, float* scores, int32_t* counts, float* max_conf,
                           int32_t* persons, void* stream);

/* SORT (lib/track/sort.py, called at lib/pose/hrnet/pose_estimation/gen_kpts.py:143,213,306) for S sequences (videos
 * or cameras) at once, K frames per call, one CTA per sequence with its frames in order.
 * gast_sort_state_bytes: the state of S sequences of at most `capacity` trackers (1 .. 4096); 0 on refusal.  Each
 *   sequence's state starts with eight int64 words: frame_count, next id, trackers, status, max_age, min_hits,
 *   capacity and a tag; the ordered tracker list and each tracker's fp64 x[7], P[7x7], id, time_since_update, hits,
 *   hit_streak and age follow.
 * gast_sort_init: Sort(max_age, min_hits) in every sequence; the first tracker of sequence s gets id first_ids[s]
 *   (device int64 (S), or null for 0), as KalmanBoxTracker.count would have it.
 * gast_sort_update: Sort.update for frame t of sequence s with the detections boxes[s, t, :counts[s, t]] ((S, K,
 *   max_det, 4) float32, person_boxes' layout; counts (S, K) int32).  out_rows (S, K, capacity, 5) float64 gets the
 *   reference's return value, [x1, y1, x2, y2, id + 1] in its order (the tracker list reversed, filtered by
 *   time_since_update < 1 and (hit_streak >= min_hits or frame_count <= min_hits)); rows past out_counts[s, t] are
 *   not written.  GAST_SORT_SKIP_EMPTY skips a frame whose count is 0 or whose boxes are all zero, as gen_video_kpts
 *   does: no update, frame_count stays, out_counts -1.  status (S) int32 gets the sequence's status word: nonzero
 *   makes its outputs from that frame on invalid (out_counts 0) and is never cleared: GAST_SORT_ST_COUNT a count
 *   above max_det (or below 0), GAST_SORT_ST_CAPACITY a tracker list beyond capacity, GAST_SORT_ST_IOU an IoU the
 *   reference refuses (a zero denominator, or NaN: linear_sum_assignment raises), GAST_SORT_ST_INF a predicted box
 *   with an infinite, non-NaN coordinate (the reference's trks and trackers go out of step), GAST_SORT_ST_STATE a
 *   state not initialised for this capacity.  The state lives in shared memory for the launch: the capacity and
 *   max_det must fit 227 KB (about 490 bytes per tracker), else the call is refused before any launch.
 * Device pointers, the caller's stream, no allocation, synchronisation or host read, so an update can be captured in
 * a graph; no atomics, calls repeat bit for bit.  Formulas in DESIGN.md §8.8. */
#define GAST_SORT_SKIP_EMPTY 1
#define GAST_SORT_ST_COUNT 1
#define GAST_SORT_ST_CAPACITY 2
#define GAST_SORT_ST_IOU 4
#define GAST_SORT_ST_INF 8
#define GAST_SORT_ST_STATE 16
size_t gast_sort_state_bytes(int32_t S, int32_t capacity);
int gast_sort_init(void* state, int32_t S, int32_t capacity, int32_t max_age, int32_t min_hits,
                   const int64_t* first_ids, void* stream);
int gast_sort_update(void* state, int32_t S, int32_t capacity, int32_t K, const float* boxes, const int32_t* counts,
                     int32_t max_det, int32_t flags, double* out_rows, int32_t* out_counts, int32_t* status,
                     void* stream);

/* SORT's tracks to the 2D pose net's crop records (lib/pose/hrnet/pose_estimation/gen_kpts.py:214-256), so that no
 * per-box host work lies between the tracker and the pose net.
 * gast_track_records: reads gast_sort_update's outputs of S sequences x K frames as they are (rows (S, K, capacity,
 *   5) float64, only rows [0, counts[s, t]) read; counts (S, K) int32, -1 a skipped frame; status (S) int32) and
 *   applies gen_video_kpts' record rule to every frame: k <= 0 tracks drop the frame, k = 1 keeps the one row,
 *   k >= num_person keeps the last num_person rows reversed (select_tracks).  Each kept box is rounded as
 *   round(v, 2), goes through box_to_center_scale with the frame's (H, W) in the model-size slots (PreProcess's call)
 *   and get_affine_transform to the out_w x out_h crop, with the reference's float32 / float64 steps, and the matrix
 *   is cv2.getAffineTransform's (OpenCV's 6 x 6 LU, unfused double; a pivot below 100 * DBL_EPSILON gives a zero
 *   matrix), bit for bit.  Record r, contiguous in (s, t, p) order over all sequences, gets frame_index[r] = s * K +
 *   t, slots[r] = t' * num_person + p (t' the frame's rank among the sequence's kept frames), forward_mats[6r..6r+5]
 *   and center_scale[4r..4r+3] = (center x, center y, scale x, scale y) float32.  The arrays must hold S * K *
 *   num_person records; those past the total are not written.  summary (S, 4) int32: the sequence's records, its kept
 *   frames, its status word and the first frame (t) that set a GAST_REC_ST_TRACKS, GAST_REC_ST_NONFINITE or
 *   GAST_REC_ST_EMPTY bit (-1 for none).  The status word is SORT's word (its low bits) or'ed with:
 *   GAST_REC_ST_TRACKS a frame with 2 .. num_person - 1 tracks (the reference's reshape raises) or a count outside
 *   -1 .. capacity, GAST_REC_ST_NONFINITE a kept box with a non-finite coordinate, GAST_REC_ST_EMPTY a kept box with
 *   a non-positive width and height (its triangle is singular), GAST_REC_ST_MATRIX a non-finite forward matrix.
 *   total (1) int32: all sequences' records.  Sides <= 32767; S * K * num_person < 2^31.
 * gast_record_inverse: get_affine_transform(center, scale, 0, (hw, hh), inv=1) of the first min(n, *total) records'
 *   center_scale (n, 4) float32 (total: a device int32, or null for n): inverse_mats (n, 6) float64, the heatmap ->
 *   frame matrices get_final_preds applies, with the same triangles and LU, bit for bit.
 * Device pointers, the caller's stream, no allocation, synchronisation or host read, so both can be captured in a
 * graph; no atomics, calls repeat bit for bit and a sequence's records do not depend on the other sequences' rows.
 * Formulas in DESIGN.md §8.9. */
#define GAST_REC_ST_TRACKS 0x100
#define GAST_REC_ST_NONFINITE 0x200
#define GAST_REC_ST_EMPTY 0x400
#define GAST_REC_ST_MATRIX 0x800
int gast_track_records(const double* rows, const int32_t* counts, const int32_t* status, int32_t S, int32_t K,
                       int32_t capacity, int32_t num_person, int32_t W, int32_t H, int32_t out_w, int32_t out_h,
                       int32_t* frame_index, int64_t* slots, double* forward_mats, float* center_scale,
                       int32_t* summary, int32_t* total, void* stream);
int gast_record_inverse(const float* center_scale, int32_t n, const int32_t* total, int32_t hw, int32_t hh,
                        double* inverse_mats, void* stream);

/* The live tick (gen_img_kpts, lib/pose/hrnet/pose_estimation/gen_kpts.py:115-175, into the causal real-time streams
 * and revise_skes_real_time) for C cameras of P = num_person slots each, one frame per camera and tick; slot p of
 * camera c is row c * P + p.  A slot is bound to a SORT id: it keeps that id's stream across ticks.
 * gast_live_slots: reads gast_sort_update's outputs of C sequences x 1 frame as they are (rows (C, capacity, 5),
 *   counts (C), sort_status (C)) and selects a frame's tracks as gen_img_kpts does (k <= 0: none, k = 1: row 0,
 *   k >= P: rows k-1 .. k-P; 2 <= k < P: none and GAST_REC_ST_TRACKS), without round(v, 2).  The slot book (3, C, P)
 *   int64 holds per slot its id (the row's fifth column, -1 none), the last tick it was selected (-1 never) and
 *   whether its stream must restart; initialise it to (-1, -1, 1).  A selected id that holds a slot keeps it; the
 *   other selected ids, in selection order, take the free slots in ascending order, then the slots not selected this
 *   tick with the oldest last tick (the lowest slot on a tie), and mark them to restart.  Per slot: slot_active (C * P)
 *   int32, and the box's geometry as gast_track_records computes it: center_scale (C * P, 4) float32, forward_mats
 *   (C * P, 6) float64 to the out_w x out_h crop and, when hw, hh > 0, inverse_mats (C * P, 6) float64 from the hw x hh
 *   heatmap (hw = hh = 0: inverse_mats is not written).  A slot is inactive, and its center, scale and forward matrix
 *   zero, when it holds no selected id, or its box is not finite or empty or its forward matrix not finite (the bit is
 *   set).  status (C, 16) int64 per camera: [0] the sticky status word (SORT's word or'ed with the GAST_REC_ST_* bits),
 *   [1] the ticks so far (the tick counter: initialise to 0), [2 + b] the tick that first set bit b < 12 (-1 none).
 *   1 <= num_person <= 32.
 * gast_live_inputs: the n = C * P slots' decoded COCO keypoints preds (n, 17, 2) and maxvals (n, 17) ->
 *   gast_h36m_coco_format's H36M keypoints, scores, keep and valid of the one frame, gast_revise_kpts' repair: kpts
 *   (n, 17, 2) and scores (n, 17); x (n, 17, 2) normalize_screen_coordinates(kpts, w = W, h = H).  active (n) uint8
 *   = slot_active and keep and valid; an inactive slot's kpts, scores and x are zero.  The stream pool's device masks
 *   fresh_mask and active_mask (copies * n int32, copies = 2 with test-time augmentation: slot s and its twin s + n)
 *   get active and (active and restart); book_fresh (n) int64 (the book's third plane) is cleared for the active slots.
 * gast_live_place: revise_skes_real_time(world[active slots of camera c], kpts[same], width) for every camera: world
 *   (n, 17, 3) camera_to_world's poses, kpts (n, 17, 2), active (n) uint8 -> out (n, 17, 3), inactive slots zero.
 * Device pointers, the caller's stream, no allocation, synchronisation or host read, so a tick can be captured in a
 * graph; no atomics, calls repeat bit for bit.  Formulas in DESIGN.md §8.10. */
int gast_live_slots(const double* rows, const int32_t* counts, const int32_t* sort_status, int32_t C, int32_t capacity,
                    int32_t num_person, int32_t W, int32_t H, int32_t out_w, int32_t out_h, int32_t hw, int32_t hh,
                    int64_t* book, int64_t* status, int32_t* slot_active, double* forward_mats, double* inverse_mats,
                    float* center_scale, void* stream);
int gast_live_inputs(const float* preds, const float* maxvals, const int32_t* slot_active, int32_t n, int32_t W,
                     int32_t H, int32_t copies, int64_t* book_fresh, float* kpts, float* scores, float* x,
                     int32_t* fresh_mask, int32_t* active_mask, uint8_t* active, void* stream);
int gast_live_place(const float* world, const float* kpts, const uint8_t* active, int32_t C, int32_t num_person,
                    double width, float* out, void* stream);

/* The delayed live tick of the non-causal models (latency = (receptive_field - 1) / 2 >= 1): each slot's stream holds
 * one person's sequence, the frames where the slot was active joined across the ticks where it was not (gen_pose over
 * valid_frames), and a push returns the pose of the frame the slot pushed latency pushes earlier.  seq (4, C * P)
 * int64 per slot: the SORT id of its current sequence (-1 none), the tick of its last push (-1 never), the frames of
 * the sequence (0: none pending) and the length of the sequence that ended this tick (0: none); initialise it to
 * (-1, -1, 0, 0).  The ring per slot holds the repaired keypoints ring_kpts (C * P, latency + 1, 17, 2) float32 and the
 * camera tick ring_ticks (C * P, latency + 1) int64 of its last latency + 1 frames; frame f of a sequence (from 0) is at
 * ring position f mod (latency + 1).
 * gast_live_delayed_inputs: gast_live_inputs' outputs (with C, num_person for n = C * P and the whole slot book (3, C,
 *   P)), and each slot's sequence at this tick (status[c, 1] - 1, after gast_live_slots): a slot's sequence ends when
 *   it pushes with the restart flag set, or, with max_gap >= 0, when it has not pushed for more than max_gap ticks; in
 *   both cases only with frames pending.  A gap end sets the restart flag, so the next push starts a new sequence
 *   (max_gap = -1: never).  tail_mask (copies * n) int32 marks the ending slots for both halves; seq[3] gets their
 *   lengths and tail_ids (n) int64 their sequences' ids (-1 elsewhere).  A push updates seq[0..2].
 * gast_live_delayed_end: every slot of a camera with cameras[c] != 0 (cameras (C) uint8 on the device) that has frames
 *   pending ends its sequence: tail_mask, seq[3] and tail_ids as above; the others get no tail.  seq[2] is left to the
 *   caller's reset.
 * gast_live_delayed_place: one CTA per camera, three groups placed as revise_skes_real_time places them, each pose with
 *   the repaired keypoints of its own frame (the ring's; this tick's kpts (n, 17, 2) for the newest frame):
 *   - final: world (n, 17, 3) the pushed poses; poses (n, 17, 3) and frame (n) int64 the camera tick of the frame they
 *     belong to, for each slot that pushed (active (n) uint8) with at least latency + 1 frames; z rebased over those
 *     slots of the camera;
 *   - provisional (lookahead L in [0, latency), -1 none): world_now (n, now_rows = latency - L, 17, 3) a peek's poses,
 *     row now_rows - 1 of every pushed slot with at least L + 1 frames, the frame L behind its newest; now and now_frame
 *     as poses and frame;
 *   - tail: world_tail (n, latency, 17, 3) a latency-row peek of the ending slots' streams before the push; row k of a
 *     slot is frame seq[3] - latency + k of its ended sequence when that is >= 0; tail (n, latency, 17, 3) and
 *     tail_frame (n, latency), each row placed on its own (z rebased over its 17 joints).
 *   Unused rows are zero and their frames -1.  Then the ring takes this tick's kpts and tick at the pushed slots' newest
 *   positions, after every read of it.  active null (after gast_live_delayed_end): only the tails are written, and
 *   world, world_now, kpts, poses, frame, now and now_frame are not read.
 * Device pointers, the caller's stream, no allocation, synchronisation or host read; no atomics, calls repeat bit for
 * bit.  Formulas in DESIGN.md §8.11. */
int gast_live_delayed_inputs(const float* preds, const float* maxvals, const int32_t* slot_active, int32_t C,
                             int32_t num_person, int32_t W, int32_t H, int32_t copies, int32_t max_gap,
                             const int64_t* status, int64_t* book, int64_t* seq, float* kpts, float* scores, float* x,
                             int32_t* fresh_mask, int32_t* active_mask, int32_t* tail_mask, uint8_t* active,
                             int64_t* tail_ids, void* stream);
int gast_live_delayed_end(const uint8_t* cameras, int32_t C, int32_t num_person, int32_t copies, int64_t* seq,
                          int32_t* tail_mask, int64_t* tail_ids, void* stream);
int gast_live_delayed_place(const float* world, const float* world_tail, const float* world_now, int32_t now_rows,
                            const float* kpts, const uint8_t* active, const int64_t* seq, const int64_t* status,
                            int32_t C, int32_t num_person, int32_t latency, int32_t lookahead, double width,
                            float* ring_kpts, int64_t* ring_ticks, float* poses, int64_t* frame, float* now,
                            int64_t* now_frame, float* tail, int64_t* tail_frame, void* stream);

/* optim.Adam(amsgrad=True) (trainval.py:78,162-164) for every parameter in one launch.  table (n_chunks,4)
 * int64 on the device: {param pointer, grad pointer, offset into the flat state buffers, count <=
 * gast_adam_chunk()}.  max_exp_avg_sq null = plain Adam.  step = 1 for the first update. */
int32_t gast_adam_chunk(void);
int gast_adam_step(const int64_t* table, int32_t n_chunks, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                   double lr, double beta1, double beta2, double eps, double weight_decay, int64_t step, void* stream);

/* ---- whole training epochs on the device (gast_b200.training.EpochTrainer) --------------------------------------
 * A training step that one CUDA graph captures once and replays for every batch of an epoch reads which batch it is
 * from a device int64 batch counter *batch (b below) that the epoch keeps: 0 at the start of the epoch, advanced by
 * gast_epoch_loss_accumulate, the last launch of a step.  None of the three reads device data on the host,
 * allocates or synchronises.
 *
 * gast_chunk_gather_indexed: gast_chunk_gather's arguments, with pairs the whole epoch's (n_pairs,4) int32 pair
 *   table; writes exactly what gast_chunk_gather writes for pairs[b*batch_stride .. b*batch_stride + B - 1], bit for
 *   bit (batch_stride >= B: the full batch size, so that a shorter last batch is served with its own B).  Writes
 *   nothing when those rows are not all in the table. */
int gast_chunk_gather_indexed(const float* poses_2d, const float* poses_3d, const float* cameras, const int64_t* seq_start,
                              int32_t n_seq, const int32_t* pairs, int64_t n_pairs, int32_t batch_stride,
                              const int64_t* batch, int32_t B, int32_t chunk, int32_t pad, int32_t causal_shift,
                              int32_t J2, int32_t F2, int32_t J3, int32_t ncam, int32_t n_sym2, const int32_t* kps_left,
                              const int32_t* kps_right, int32_t n_sym3, const int32_t* joints_left,
                              const int32_t* joints_right, float* batch_2d, float* batch_3d, float* batch_cam,
                              void* stream);

/* gast_adam_step_table: coef (2*n_steps) (host) receives, for steps first_step .. first_step + n_steps - 1,
 *   {lr / bc1, sqrt(bc2)} computed and rounded to float exactly as gast_adam_step computes them (in double, C pow).
 * gast_adam_step_indexed: gast_adam_step at step first_step + b, with coef (2*n_steps) that table on the device:
 *   bit for bit the same update.  No update when b >= n_steps. */
int gast_adam_step_table(double lr, double beta1, double beta2, int64_t first_step, int32_t n_steps, float* coef);
int gast_adam_step_indexed(const int64_t* table, int32_t n_chunks, float* exp_avg, float* exp_avg_sq,
                           float* max_exp_avg_sq, double beta1, double beta2, double eps, double weight_decay,
                           const float* coef, int64_t n_steps, const int64_t* batch, void* stream);

/* gast_epoch_loss_accumulate: losses[b] = *loss (when b < n_steps), *sum += (double)weight * (double)*loss (fp64),
 *   then *batch = b + 1.  With weight = B * T_out of the step, *sum / (sum of the weights) is main.train's epoch
 *   loss (main.py:231,242) bit for bit. */
int gast_epoch_loss_accumulate(const float* loss, int64_t weight, double* sum, float* losses, int64_t n_steps,
                               int64_t* batch, void* stream);

/* Test/probe entry (not on the forward path): out[M,N] = A[M,K] . W[N,K]^T on one GEMM core
 * (core 0 = tensor cores, tc_mode 0 = fp32-grade as inference runs it, three scaled fp16 products (F16X3),
 * 1 = single-pass TF32, 3 = fp32-grade as training runs it, three TF32 products (3xTF32), or 16 = the half form of
 * gast_set_activation_dtype(h, GAST_F16): A and out hold __half values, W float32; every other tc_mode is refused;
 * core 1 = FFMA, tc_mode 0).  Runs once, then `reps` timed launches
 * (CUDA events) whose mean duration is written to *ms_out (host).  Synchronises the stream. */
int gast_debug_gemm(const float* A, const float* W, float* out, int32_t M, int32_t N, int32_t K,
                    int32_t core, int32_t tc_mode, int32_t reps, float* ms_out, void* stream);

/* Test/probe entry (not on the training path): dW[N,K] = dZ[M,N]^T . A[M,K] (dense row-major operands) as the
 * training backward computes a weight gradient: the same row splits on this device, one contraction kernel over
 * them, the fixed-order reduction of the partials.  core 1 = the FFMA kernel (exact fp32, tc_mode 0); core 0 with
 * tc_mode 1 = the kernel TF32 training runs: the TF32 tensor-core kernel where N % 32 == 0, K % 32 == 0 and dZ is
 * 16-byte aligned, the FFMA kernel elsewhere.
 * core 0 with tc_mode 0 fails: there is no fp32-grade tensor-core weight gradient.  Runs once, then `reps` timed
 * runs whose mean duration (contraction + reduction) is written to *ms_out (host).  Synchronises the stream. */
int gast_debug_wgrad(const float* dZ, const float* A, float* dW, int32_t M, int32_t N, int32_t K,
                     int32_t core, int32_t tc_mode, int32_t reps, float* ms_out, void* stream);

/* Test-only audit of every GEMM launch a handle makes (forward, training, gradients, chunked calls, streams).
 * A plain-C mirror of the launch's parameters: the rows of A come from up to three K-segments, output row
 * f J + j of segment s reading source row (map_s(f) J + j) at base_s + row ld_s + tap tap_stride_s + c for column
 * tap Kc_s + c of the segment, map(f) = (f / T_out) T_in + (f % T_out) t_mul + t_off.  W is [N][ldw] K-major, the
 * output [F J][ld_out].  epi 0 (plain): relu?(A W^T + bias) + res[(res_map(f) J + j) res_ld]; 1 (SemCH): per 128
 * columns of W (mask = tile / tiles_per_mask), 64 self and 64 neighbour products mixed over nbr[mask] with coef
 * [nnz][C] and shift [2][C] into columns mask C + c; 2 (global attention): softmax over joints of
 * LeakyReLU_0.2(ab[i, 2h] + ab[j, 2h + 1]) + ck[h][i][j] mixing G = A W^T + bg, head h = column / Cg. */
typedef struct gast_gemm_audit_seg {
  const float* base;
  int64_t tap_stride;                    /* floats added per tap */
  int32_t ld, K, Kc;                     /* row stride, columns (taps * Kc), columns per tap */
  int32_t T_out, T_in, t_mul, t_off;     /* frame map */
} gast_gemm_audit_seg;

typedef struct gast_gemm_audit {
  int64_t index;                         /* running index of the handle's audited launches */
  int32_t epi;                           /* 0 plain, 1 SemCH, 2 global attention */
  int32_t core;                          /* the core that runs: 0 tensor cores, 1 FFMA */
  int32_t tc_form;                       /* tensor cores: 0 3xTF32, 1 1xTF32, 2 F16X3, 3 half (A, out, res fp16); FFMA: -1 */
  int32_t tma_mask;                      /* tensor cores: bit s set when segment s is fed by TMA */
  int32_t nseg;
  gast_gemm_audit_seg seg[3];
  const float* W;
  int32_t ldw, N, F, J, fpt, ld_out;
  float* out;
  const float* bias;
  int32_t relu, res_ld;
  const float* res;
  int32_t res_T_out, res_T_in, res_t_mul, res_t_off;
  const float* coef[2];                  /* SemCH */
  const float* shift;
  int32_t C, tiles_per_mask;
  uint8_t nbr_row_ptr[2][36];            /* neighbours of joint i: nbr_col[m][row_ptr[m][i] .. row_ptr[m][i + 1]) */
  uint8_t nbr_col[2][164];
  const float* ab;                       /* global attention */
  const float* ck;
  const float* bg;
  int32_t heads, Cg;
} gast_gemm_audit;

/* fn(0, d, user) runs just before a launch and fn(1, d, user) just after it, the stream synchronised before each
 * call, so that fn may read every operand and the output.  A non-zero return fails the call.  fn == NULL turns the
 * audit off; a launch into a stream under CUDA-graph capture is not audited and is counted instead
 * (gast_debug_gemm_audit_skips). */
typedef int (*gast_gemm_audit_fn)(int32_t phase, const gast_gemm_audit* d, void* user);
int gast_debug_set_gemm_audit(gast_t* h, gast_gemm_audit_fn fn, void* user);
int64_t gast_debug_gemm_audit_skips(const gast_t* h);

/* Test-only audit of the other kernels of the inference forward and the streams, on the GEMM audit's terms: every
 * launch of the expand, the theta/phi row dots (the training forward's too), the attention mix kernel and the shrink.
 *   expand (kind 0):  out[r][c] = relu(be[c] + sum_{kk < taps, i < Fin} We[kk Fin + i][c] x[((b T + t stride + kk) J + j)
 *                     Fin + i]) for rows r = (b T0 + t) J + j < rows, c < C = K (ld = C); variant = KFT (6 or 10).
 *   rowdot (1):       ab[r][q] = X[r ld + k] U[q][k] + cab[q], q < Q = 2 heads, k < K; variant 0 = rowdot8_kernel,
 *                     else Q of rowdot_kernel<Q>; block = the handle's graph-attention block.
 *   mix (2):          Y[(f J + i) ld + n] = sum_j att_{n / Cg}[f, i, j] G[(f J + j) ld + n], n < heads Cg, f < F, with
 *                     att_h = softmax_j(LeakyReLU_0.2(ab[f J + i][2h] + ab[f J + j][2h + 1])) + Ck[h][i][j]; fpb frames
 *                     per CTA; block as for rowdot.
 *   shrink (3):       out[r][o] = X[r ld + k] Ws[o][k], o < 3, k < K.
 *   shrink_mpjpe (4): shrink into out, and *loss = mean_r ||out[r] - target[r]||.
 * in_type / out_type: 0 float32, 1 fp16 (the rowdot's ab and shrink_mpjpe's out, target and loss are float32).
 * gemm_index: the number of GEMM launches the GEMM audit had checked before this one. */
typedef struct gast_kernel_audit {
  int64_t index;                         /* running index of the handle's audited kernel launches */
  int64_t gemm_index;
  int32_t kind;                          /* 0 expand, 1 rowdot, 2 mix, 3 shrink, 4 shrink_mpjpe */
  int32_t variant, fpb, block;
  int32_t in_type, out_type;
  const void* x;                         /* x (expand), X (rowdot, shrink) or G (mix) */
  const float* We; const float* be;      /* expand */
  const float* U; const float* cab;      /* rowdot */
  float* ab;                             /* rowdot: written; mix: read */
  const float* Ck;                       /* mix */
  const float* Ws; const float* target;  /* shrink */
  float* loss;
  void* out;                             /* out (expand, shrink) or Y (mix) */
  int64_t rows;                          /* rows (expand, rowdot, shrink) or frames F (mix) */
  int32_t K, ld, J, T, T0, stride, taps, Fin, heads, Cg;
} gast_kernel_audit;

typedef int (*gast_kernel_audit_fn)(int32_t phase, const gast_kernel_audit* d, void* user);
int gast_debug_set_kernel_audit(gast_t* h, gast_kernel_audit_fn fn, void* user);
int64_t gast_debug_kernel_audit_skips(const gast_t* h);

const char* gast_last_error(void);
const char* gast_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GAST_B200_H */
