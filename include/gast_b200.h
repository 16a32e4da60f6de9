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
 * precision).  Not a fallback switch: both are CUDA paths. */
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
 * Any other value fails.  Everything else (expand, row-dots, the attention mix, shrink, GEMMs the tensor-core core
 * does not take, every GEMM under gast_set_gemm_core(h, 1)) stays fp32.  Like a core switch it needs no
 * gast_prepare, costs nothing and does not invalidate stream `state`. */
int gast_set_precision(gast_t* h, int32_t mode);

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
 *   here; gast_b200.realtime.CausalStream refuses such a push.  gast_set_gemm_core and gast_set_precision do not
 *   invalidate `state`. */
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
 *   snapshot does not depend on the ring phase.
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
 * (:51-59), 2 = coco_h36m_toe_format (T,J_in>=22,2)->(T,19,2) (:62-78).  valid (T) int32, may be null:
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

/* common/loss.py:5-11 mpjpe: *loss = mean_i ||pred_i - target_i|| over n_points rows of D (<= 4) coordinates;
 * when dpred is not null it receives grad_scale * d loss / d pred (the backward of the same pass).
 * workspace: gast_mpjpe_workspace_bytes() bytes of scratch. */
size_t gast_mpjpe_workspace_bytes(void);
int gast_mpjpe(const float* pred, const float* target, int64_t n_points, int32_t D, float* loss, float* dpred,
               float grad_scale, void* workspace, void* stream);

/* common/loss.py:14-53 p_mpjpe: per_frame[n] = mean joint distance of frame n after the similarity
 * (Procrustes) alignment of pred[n] (J,3) to target[n]; the reference's scalar is the mean of per_frame. */
int gast_p_mpjpe(const float* pred, const float* target, int32_t N, int32_t J, float* per_frame, void* stream);

/* optim.Adam(amsgrad=True) (trainval.py:78,162-164) for every parameter in one launch.  table (n_chunks,4)
 * int64 on the device: {param pointer, grad pointer, offset into the flat state buffers, count <=
 * gast_adam_chunk()}.  max_exp_avg_sq null = plain Adam.  step = 1 for the first update. */
int32_t gast_adam_chunk(void);
int gast_adam_step(const int64_t* table, int32_t n_chunks, float* exp_avg, float* exp_avg_sq, float* max_exp_avg_sq,
                   double lr, double beta1, double beta2, double eps, double weight_decay, int64_t step, void* stream);

/* Test/probe entry (not on the forward path): out[M,N] = A[M,K] . W[N,K]^T on one GEMM core
 * (core 0 = tensor cores, tc_mode 0 = fp32-grade as inference runs it, three scaled fp16 products (F16X3),
 * 1 = single-pass TF32, or 3 = fp32-grade as training runs it, three TF32 products (3xTF32); tc_mode 2 is not a
 * mode and is refused; core 1 = FFMA, tc_mode 0).  Runs once, then `reps` timed launches
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

const char* gast_last_error(void);
const char* gast_version(void);

#ifdef __cplusplus
}
#endif
#endif /* GAST_B200_H */
