"""Frame-by-frame lifting of many concurrent keypoint streams (SURVEY.md §8f N4).

The reference's real-time model is a causal `SpatioTemporalModelOptimized1f` fed the last `receptive_field`
frames of one stream for every new frame (`gen_skes.py:43-69`, `tools/inference.py:19-110`): O(rf) work per
frame.  `PoseStream` produces the same poses with O(1) work per frame: the library keeps, per temporal stage, a
ring of that stage's past inputs for all streams (`csrc/stream.cuh`, C ABI `gast_stream_push_ex`), so a pushed frame
computes one new position per layer.  A stream's first frame stands for its whole (edge-padded) history exactly
like `UnchunkedGenerator` does (`common/generators.py:210-221`).

`PoseStream` takes causal and non-causal models.  A non-causal model returns the pose of frame t - pad when frame t
is pushed (`latency` = pad = (rf - 1) // 2; 0 for a causal model).  `end()` closes a stream's sequence: its next
`latency` pushes repeat the last frame (the generator's right padding) and return the remaining poses.  With
`augment=True` every push also runs the mirrored twin and averages it back, as every inference helper of the
reference does (`tools/inference.py:19-110`).  The poses of a sequence then equal
`UnchunkedGenerator([seq], pad, causal_shift, augment)` + `tools/inference.evaluate`.  `CausalStream` is the causal,
un-augmented restriction that returns the pose of the newest frame.

The rings hold activations computed with the weights of the pushes that wrote them.  Any change to the model's
parameters or buffers (`load_state_dict`, an optimiser step, a training forward, which moves the BatchNorm running
statistics) therefore invalidates the history of every stream: the next push raises `GastError` unless `reset()`
(every stream) was called after the change.  Switching the GEMM core (`engine.set_gemm_core`) or the precision
(`engine.set_precision`, which the streams follow like every forward) changes no weight and keeps the streams.

`WindowStream` is the generic form for any callable network: a device ring of the last `rf` input frames and one
window forward per pushed frame (what the reference does; used for non-GAST callables and as the cross-check).
"""
import ctypes as C
import numpy as np
import torch

from . import _lib as L

# left/right keypoint and joint lists of the reference's inference helpers (tools/inference.py:14-15) and of
# reconstruction.py:get_joints_info for 19 joints (reconstruction.py:185 uses the same lists for the keypoints)
SYMMETRY = {
    17: ([4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]),
    19: ([5, 6, 7, 8, 13, 14, 15], [1, 2, 3, 4, 16, 17, 18]),
}


class SequenceBook(object):
    """Host-side sequence bookkeeping of `n` streams with output latency `latency` (no CUDA, no device sync).

    A stream is LIVE (its pushes append frames to its current sequence), ENDING (`end` was called: its next pushes
    are held and return the sequence's last poses) or IDLE (held, nothing due).  `advance()` is called once per push
    and returns the fresh and hold masks of that push and, per stream, the position within the current sequence of
    the frame whose pose that push returns (-1 where nothing is due)."""

    def __init__(self, n, latency):
        self.n, self.latency = int(n), int(latency)
        self.fresh = np.ones(self.n, dtype=bool)            # the next push starts a new sequence
        self.length = np.zeros(self.n, dtype=np.int64)      # frames in the current sequence
        self.left = np.full(self.n, -1, dtype=np.int64)     # -1 live; k >= 0: k held pushes left (0 = idle)

    def _sel(self, streams):
        if streams is None:
            return slice(None)
        return np.asarray(streams, dtype=np.int64).reshape(-1)

    def reset(self, streams=None):
        s = self._sel(streams)
        self.fresh[s] = True
        self.length[s] = 0
        self.left[s] = -1

    def end(self, streams=None):
        s = np.arange(self.n)[self._sel(streams)]
        s = s[self.left[s] < 0]                           # already ending or idle: nothing to do
        empty = self.fresh[s]                             # reset but nothing pushed since: an empty sequence
        self.fresh[s[empty]] = False
        self.left[s[empty]] = 0
        self.left[s[~empty]] = self.latency

    def all_restarting(self):
        """every stream either starts anew at the next push or is idle (its history is never read again)"""
        return bool(np.all(self.fresh | (self.left == 0)))

    def advance(self):
        """-> (fresh, hold, index) of the next push; updates the state as that push does"""
        fresh = self.fresh.copy()
        self.length[fresh] = 0
        self.left[fresh] = -1
        live = self.left < 0
        hold = ~live
        index = np.full(self.n, -1, dtype=np.int64)
        index[live] = self.length[live] - self.latency
        self.length[live] += 1
        ending = self.left > 0
        # the k-th held push (k = latency - left + 1) returns frame length - 1 + k - latency
        index[ending] = self.length[ending] - self.left[ending]
        self.left[ending] -= 1
        index[index < 0] = -1
        self.fresh[:] = False
        return fresh, hold, index

    def advance_many(self, K, valid=None):
        """-> (fresh (n,), hold (n, K), index (n, K)) of K consecutive pushes, as K calls of `advance()` return them,
        with `end([s])` before push valid[s] of every live stream s whose valid[s] < K (0 <= valid[s] <= K; None:
        no end).  Vectorised over the pushes: every stream is live up to its end and held from then on."""
        K = int(K)
        if K < 1:
            raise ValueError('advance_many: K must be at least 1 (got %d)' % K)
        if valid is None:
            e = np.full(self.n, K, dtype=np.int64)
        else:
            e = np.asarray(valid, dtype=np.int64).reshape(-1)
            if e.shape != (self.n,) or (e < 0).any() or (e > K).any():
                raise ValueError('advance_many: valid must hold %d values in [0, %d]' % (self.n, K))
        live = self.left < 0                               # live at the first push (a fresh stream is live)
        ends = live & (e < K)
        empty = ends & self.fresh & (e == 0)               # ended before its first frame: idle at once
        # the held part of every stream starts at push kh with `left0` pushes left and a sequence of `lh` frames
        kh = np.where(live, e, 0)
        left0 = np.where(live, np.where(empty, 0, self.latency), self.left)
        len0 = np.where(self.fresh, 0, self.length)
        lh = np.where(live, len0 + kh, self.length)
        k = np.arange(K, dtype=np.int64)[None, :]
        hold = k >= kh[:, None]
        index = np.where(hold, -1, len0[:, None] + k - self.latency)
        left_k = left0[:, None] - (k - kh[:, None])        # pushes left before each held push
        due = hold & (left_k > 0)
        index[due] = (lh[:, None] - left_k)[due]
        index[index < 0] = -1
        fresh = self.fresh & ~empty
        self.length = lh
        self.left = np.where(live & ~ends, -1, np.maximum(left0 - (K - kh), 0))
        self.fresh[:] = False
        return fresh, hold, index


class PoseStream(object):
    """O(1)-per-frame lifting of `n_streams` concurrent streams with any non-dense model of the drop-in classes
    (`SpatioTemporalModel` or `SpatioTemporalModelOptimized1f`, causal or not: the weights are interchangeable).

    push(frame (n, J, F)) -> (poses (n, J, 3) CUDA, index (n,) CPU int64): poses[s] is the pose of frame index[s] of
    stream s's current sequence, or unspecified where index[s] == -1.  The kps/joints lists default to the
    reference's for J = 17 and J = 19; `augment=True` with another J needs all four."""

    def __init__(self, model_pos, n_streams, augment=False, kps_left=None, kps_right=None, joints_left=None,
                 joints_right=None, device=None):
        from . import engine
        name = type(self).__name__
        if not hasattr(model_pos, '_gast_causal'):
            raise engine.GastError('%s needs a model of the drop-in classes (model/gast_net.py)' % name)
        if getattr(model_pos, '_gast_dense', False):
            raise engine.GastError('%s: the dense ablation has no streaming form' % name)
        if device is None:
            device = next(model_pos.parameters()).device
        self.device = torch.device(device)
        if self.device.type != 'cuda':
            raise engine.GastError('%s: the model must be on a CUDA device (there is no CPU path)' % name)
        self.model = model_pos
        self.engine = engine
        self.rf = int(model_pos.receptive_field())
        self.n = int(n_streams)
        self.J = int(model_pos.num_joints_in)
        self.F = int(model_pos.in_features)
        self.causal = bool(model_pos._gast_causal)
        self.latency = 0 if self.causal else (self.rf - 1) // 2
        self.augment = bool(augment)
        if self.augment:
            lists = [kps_left, kps_right, joints_left, joints_right]
            if any(v is None for v in lists):
                if self.J not in SYMMETRY:
                    raise engine.GastError('%s: augment=True with %d joints needs kps_left, kps_right, joints_left and '
                                           'joints_right (defaults exist for 17 and 19 joints)' % (name, self.J))
                left, right = SYMMETRY[self.J]
                lists = [d if v is None else v for v, d in zip(lists, [left, right, left, right])]
            self.kps_left, self.kps_right, self.joints_left, self.joints_right = [[int(i) for i in v] for v in lists]
            if len(self.kps_left) != len(self.kps_right) or len(self.joints_left) != len(self.joints_right):
                raise engine.GastError('%s: left and right lists differ in length' % name)
            arr = lambda v: (C.c_int32 * len(v))(*v)   # noqa: E731
            self._kl, self._kr = arr(self.kps_left), arr(self.kps_right)
            self._jl, self._jr = arr(self.joints_left), arr(self.joints_right)
        self.copies = 2 if self.augment else 1      # streams the library runs: [original | mirrored]
        self.book = SequenceBook(self.n, self.latency)
        self.step = 0
        self._masks = torch.zeros((2, self.copies * self.n), dtype=torch.int32, device=self.device)
        self._sig = None                 # the handle's parameter signature at the last push
        self._state = None
        self._ws = None
        self._chunk_ws = None            # push_frames: workspace of the largest K so far
        self._chunk_masks = None

    def reset(self, streams=None):
        """Start new sequences on all (or the listed) streams with the next pushed frame; drop any pending tail."""
        self.book.reset(streams)

    def end(self, streams=None):
        """The current sequences of all (or the listed) streams ended with their last pushed frame.  Their next
        `latency` pushes ignore the caller's rows and return the remaining poses; then they are idle until reset."""
        self.book.end(streams)

    def _upload(self, fresh, hold):
        """-> device pointers of the fresh and hold masks of this push (None where no stream is set)"""
        any_f, any_h = bool(fresh.any()), bool(hold.any())
        if not (any_f or any_h):
            return None, None
        mk = np.tile(np.stack([fresh, hold]).astype(np.int32), (1, self.copies))
        # pinned + non_blocking: no device sync; the caching host allocator keeps the buffer until the copy ran
        self._masks.copy_(torch.from_numpy(mk).pin_memory(), non_blocking=True)
        return (self._masks[0].data_ptr() if any_f else None), (self._masks[1].data_ptr() if any_h else None)

    def _begin(self, h, st):
        """refresh the handle, refuse a push over history computed with other weights, allocate the state"""
        eng, lib = self.engine, h.lib
        h.refresh(self.model, st)
        if self._sig is not None and h.sig != self._sig and not self.book.all_restarting():
            raise eng.GastError('%s: the model\'s parameters or buffers changed since the last push '
                                '(load_state_dict, an optimiser step or a training forward); the streams\' history '
                                'was computed with the old weights -- call reset() before pushing again'
                                % type(self).__name__)
        if self._state is None:
            m = self.copies * self.n
            if lib.gast_stream_latency(h.h) != self.latency:
                raise eng.GastError('gast_stream_latency: %s' % L.last_error())
            nb = lib.gast_stream_state_bytes(h.h, m)
            wb = lib.gast_stream_workspace_bytes(h.h, m)
            if nb == 0 or wb == 0:
                raise eng.GastError('gast_stream_state_bytes: %s' % L.last_error())
            self._state = torch.empty(int(nb), dtype=torch.uint8, device=self.device)
            self._ws = torch.empty(int(wb), dtype=torch.uint8, device=self.device)

    def push(self, frame):
        """frame (n_streams, J, in_features): the newest 2D keypoints of every stream (normalised screen
        coordinates; rows of held streams are ignored) -> (poses (n, J, 3), index (n,) CPU int64)."""
        eng = self.engine
        name = type(self).__name__
        frame = torch.as_tensor(frame, dtype=torch.float32, device=self.device).contiguous()
        assert frame.shape == (self.n, self.J, self.F), frame.shape
        if self.model.training:
            raise eng.GastError('%s: call .eval() on the model (streaming is inference)' % name)
        h = eng.model_handle(self.model, self.device)
        lib = h.lib
        m = self.copies * self.n
        y = torch.empty((self.n, self.J, 3), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            self._begin(h, st)
            fresh, hold, index = self.book.advance()
            fresh_p, hold_p = self._upload(fresh, hold)
            x, out = frame, y
            if self.augment:
                x = torch.empty((2, self.n, self.J, self.F), dtype=torch.float32, device=self.device)
                if lib.gast_tta_prepare(C.c_void_p(frame.data_ptr()), C.c_void_p(x.data_ptr()), self.n, self.J, self.F,
                                        0, 0, len(self.kps_left), self._kl, self._kr, C.c_void_p(st)) != 0:
                    raise eng.GastError('gast_tta_prepare: %s' % L.last_error())
                out = torch.empty((2, self.n, self.J, 3), dtype=torch.float32, device=self.device)
            rc = lib.gast_stream_push_ex(h.h, C.c_void_p(self._state.data_ptr()), C.c_int64(self.step),
                                         C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), m, C.c_void_p(fresh_p),
                                         C.c_void_p(hold_p), C.c_void_p(self._ws.data_ptr()), self._ws.numel(),
                                         C.c_void_p(st))
            if rc != 0:
                raise eng.GastError('gast_stream_push_ex: %s' % L.last_error())
            launches = int(lib.gast_last_launch_count(h.h))
            if self.augment:
                if lib.gast_tta_merge(C.c_void_p(out.data_ptr()), C.c_void_p(y.data_ptr()), self.n, self.J,
                                      len(self.joints_left), self._jl, self._jr, C.c_void_p(st)) != 0:
                    raise eng.GastError('gast_tta_merge: %s' % L.last_error())
                launches += 2
            self._sig = h.sig
        self.step += 1
        self.last_launches = launches
        return y, torch.from_numpy(index)

    def push_frames(self, frames, valid=None):
        """frames (n_streams, K, J, in_features): the next K frames of every stream -> (poses (n, K, J, 3) CUDA,
        index (n, K) CPU int64), what K calls of `push` with frames[:, k] return, in one library call
        (gast_stream_push_chunk).  valid (n,) or None: only the first valid[s] frames of stream s belong to its
        sequence; a smaller value than K ends the sequence there (as `end([s])` before frame valid[s] would) and the
        rest of the chunk returns its tail.  Rows of held frames are ignored.  `reset()` / `end()` take effect at
        frame 0 of the call, as for `push`."""
        eng = self.engine
        name = type(self).__name__
        frames = torch.as_tensor(frames, dtype=torch.float32, device=self.device).contiguous()
        assert frames.dim() == 4 and frames.shape[0] == self.n and frames.shape[1] >= 1 and \
            tuple(frames.shape[2:]) == (self.J, self.F), frames.shape
        K = int(frames.shape[1])
        if K == 1 and valid is None:
            y, index = self.push(frames[:, 0])
            return y.view(self.n, 1, self.J, 3), index.view(self.n, 1)
        if self.model.training:
            raise eng.GastError('%s: call .eval() on the model (streaming is inference)' % name)
        h = eng.model_handle(self.model, self.device)
        lib = h.lib
        m = self.copies * self.n
        y = torch.empty((self.n, K, self.J, 3), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            self._begin(h, st)
            wb = int(lib.gast_stream_chunk_workspace_bytes(h.h, m, K))
            if wb == 0:
                raise eng.GastError('gast_stream_chunk_workspace_bytes: %s' % L.last_error())
            if self._chunk_ws is None or self._chunk_ws.numel() < wb:   # grows with K: serves every smaller K
                self._chunk_ws = None
                self._chunk_ws = torch.empty(wb, dtype=torch.uint8, device=self.device)
            fresh, hold, index = self.book.advance_many(K, valid)
            fresh_p, hold_p = self._upload_chunk(fresh, hold)
            x, out = frames, y
            if self.augment:
                # (2, n*K, J, F) = 2n streams of K frames: [original | mirrored]
                x = torch.empty((2, self.n, K, self.J, self.F), dtype=torch.float32, device=self.device)
                if lib.gast_tta_prepare(C.c_void_p(frames.data_ptr()), C.c_void_p(x.data_ptr()), self.n * K, self.J,
                                        self.F, 0, 0, len(self.kps_left), self._kl, self._kr, C.c_void_p(st)) != 0:
                    raise eng.GastError('gast_tta_prepare: %s' % L.last_error())
                out = torch.empty((2, self.n, K, self.J, 3), dtype=torch.float32, device=self.device)
            rc = lib.gast_stream_push_chunk(h.h, C.c_void_p(self._state.data_ptr()), C.c_int64(self.step),
                                            C.c_void_p(x.data_ptr()), C.c_void_p(out.data_ptr()), m, K,
                                            C.c_void_p(fresh_p), C.c_void_p(hold_p),
                                            C.c_void_p(self._chunk_ws.data_ptr()), self._chunk_ws.numel(),
                                            C.c_void_p(st))
            if rc != 0:
                raise eng.GastError('gast_stream_push_chunk: %s' % L.last_error())
            launches = int(lib.gast_last_launch_count(h.h))
            if self.augment:
                if lib.gast_tta_merge(C.c_void_p(out.data_ptr()), C.c_void_p(y.data_ptr()), self.n * K, self.J,
                                      len(self.joints_left), self._jl, self._jr, C.c_void_p(st)) != 0:
                    raise eng.GastError('gast_tta_merge: %s' % L.last_error())
                launches += 2
            self._sig = h.sig
        self.step += K
        self.last_launches = launches
        return y, torch.from_numpy(index)

    def _upload_chunk(self, fresh, hold):
        """-> device pointers of the fresh (n) and hold (n, K) masks of a chunk, repeated for the mirrored half
        (None where no stream is set)"""
        any_f, any_h = bool(fresh.any()), bool(hold.any())
        if not (any_f or any_h):
            return None, None
        m = self.copies * self.n
        mk = np.concatenate([np.tile(fresh.astype(np.int32), self.copies),
                             np.tile(hold.astype(np.int32), (self.copies, 1)).reshape(-1)])
        # kept until the next chunk, so that no allocation of this one reuses it before the push read it
        self._chunk_masks = dev = torch.empty(mk.size, dtype=torch.int32, device=self.device)
        # pinned + non_blocking: no device sync; the caching host allocator keeps the buffer until the copy ran
        dev.copy_(torch.from_numpy(mk).pin_memory(), non_blocking=True)
        return (dev.data_ptr() if any_f else None), (dev[m:].data_ptr() if any_h else None)


class CausalStream(PoseStream):
    """O(1)-per-frame lifting of `n_streams` concurrent streams with a causal model of the drop-in classes
    (`SpatioTemporalModelOptimized1f(causal=True)` as gen_skes.load_model_realtime builds it, or the dilated
    `SpatioTemporalModel(causal=True)`: the weights are interchangeable).  `push` returns the pose of the pushed
    frame of every stream: `PoseStream` without augmentation, poses only."""

    def __init__(self, model_pos, n_streams, device=None):
        from . import engine
        if not getattr(model_pos, '_gast_causal', False):
            raise engine.GastError('CausalStream needs a causal model (gen_skes.py:59 builds it with causal=True)')
        super(CausalStream, self).__init__(model_pos, n_streams, device=device)

    def push(self, frame):
        """frame (n_streams, J, in_features): the newest 2D keypoints of every stream (normalised screen
        coordinates).  Returns the 3D pose of that frame, (n_streams, J, 3)."""
        return super(CausalStream, self).push(frame)[0]

    def push_frames(self, frames):
        """frames (n_streams, K, J, in_features): the next K frames of every stream -> their 3D poses
        (n_streams, K, J, 3), what K calls of `push` return, in one library call."""
        return super(CausalStream, self).push_frames(frames)[0]


def lift_sequences(model_pos, sequences, n_streams=64, chunk=256, augment=False, kps_left=None, kps_right=None,
                   joints_left=None, joints_right=None):
    """Whole-sequence lifting in bounded memory: sequences [(T_i, J, in_features)] -> [(T_i, J, 3) CUDA tensors],
    the poses `UnchunkedGenerator` + the model forward (+ the TTA merge with `augment=True`) compute for each
    sequence, i.e. what `tta.evaluate_sequence` returns.  The sequences are packed onto `n_streams` streams of a
    `PoseStream` and pushed `chunk` frames at a time; a stream starts its next sequence at the first chunk after the
    last pose of its previous one.  The library's scratch memory depends on (n_streams, chunk), not on T_i."""
    from . import engine
    dev = next(model_pos.parameters()).device
    seqs = [torch.as_tensor(s, dtype=torch.float32).to(dev) for s in sequences]
    J, F = int(model_pos.num_joints_in), int(model_pos.in_features)
    for s in seqs:
        if s.dim() != 3 or tuple(s.shape[1:]) != (J, F):
            raise engine.GastError('lift_sequences: every sequence must be (T, %d, %d), got %s' % (J, F, tuple(s.shape)))
    lengths = [int(s.shape[0]) for s in seqs]
    starts = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    out = torch.empty((int(starts[-1]), J, 3), dtype=torch.float32, device=dev)
    todo = [q for q, T in enumerate(lengths) if T > 0]
    if todo:
        model_pos.eval()
        allx = torch.cat([seqs[q] for q in todo])                 # every frame, for one gather per chunk
        base = np.zeros(len(lengths), dtype=np.int64)             # first row of sequence q in allx
        base[todo] = np.concatenate([[0], np.cumsum([lengths[q] for q in todo])[:-1]])
        n = max(1, min(int(n_streams), len(todo)))
        ps = PoseStream(model_pos, n, augment=augment, kps_left=kps_left, kps_right=kps_right,
                        joints_left=joints_left, joints_right=joints_right, device=dev)
        lat = ps.latency
        T = np.array(lengths, dtype=np.int64)
        cur = np.full(n, -1, dtype=np.int64)                      # sequence on each stream (-1: none)
        pushed = np.zeros(n, dtype=np.int64)                      # its frames pushed so far
        steps = np.zeros(n, dtype=np.int64)                       # pushes since it started: T + latency in all
        queue = list(reversed(todo))
        with torch.no_grad():
            while True:
                for s in range(n):
                    if cur[s] < 0 or steps[s] == T[cur[s]] + lat:
                        cur[s] = -1
                        if queue:
                            cur[s], pushed[s], steps[s] = queue.pop(), 0, 0
                            ps.reset([s])
                active = cur >= 0
                if not active.any():
                    break
                Ta = T[cur[active]]
                K = int(min(chunk, (Ta + lat - steps[active]).max()))
                valid = np.zeros(n, dtype=np.int64)
                valid[active] = np.minimum(K, Ta - pushed[active])
                k = np.arange(K)[None, :]
                rows = np.where(k < valid[:, None], (base[cur.clip(min=0)] + pushed)[:, None] + k, 0)
                frames = allx[torch.from_numpy(rows).to(dev)]       # rows of held frames: any frame, not read
                y, index = ps.push_frames(frames, valid=valid)
                index = index.numpy()
                for s in np.flatnonzero(active):
                    sel = np.flatnonzero(index[s] >= 0)           # one run of consecutive poses of the sequence
                    if sel.size:
                        a, c, q = int(index[s, sel[0]]), sel.size, cur[s]
                        out[starts[q] + a:starts[q] + a + c] = y[s, sel[0]:sel[0] + c]
                    pushed[s] += valid[s]
                    steps[s] = min(steps[s] + K, T[cur[s]] + lat)
                    if pushed[s] == T[cur[s]] and valid[s] == K:
                        ps.end([s])                               # the sequence ended with the chunk's last frame
    return [out[starts[q]:starts[q + 1]] for q in range(len(lengths))]


class WindowStream(object):
    """Generic frame-by-frame driver for any window network `net((n, rf, J, F)) -> (n, T_out, J, 3)`: keeps the last
    `rf` frames of `n_streams` streams in one device tensor used as a ring and runs one window forward per pushed
    frame (O(rf) per frame, as the reference's real-time loop does)."""

    def __init__(self, net, n_streams, device=None):
        self.model = net
        self.rf = int(net.receptive_field())
        if device is None:
            device = next(net.parameters()).device
        self.device = torch.device(device)
        self.n = int(n_streams)
        self.J = int(net.num_joints_in)
        self.F = int(net.in_features)
        # ring[:, (head + k) % rf] is the k-th oldest frame of the window; `window` is its unrolled copy
        self.ring = torch.zeros((self.n, self.rf, self.J, self.F), dtype=torch.float32, device=self.device)
        self.window = torch.empty_like(self.ring)
        self.head = 0
        self.started = torch.zeros(self.n, dtype=torch.bool, device=self.device)

    def reset(self, streams=None):
        if streams is None:
            self.started.zero_()
        else:
            self.started[torch.as_tensor(streams, device=self.device)] = False

    def push(self, frame):
        frame = torch.as_tensor(frame, dtype=torch.float32, device=self.device)
        assert frame.shape == (self.n, self.J, self.F), frame.shape
        fresh = ~self.started
        if bool(fresh.any()):
            # a stream's first frame fills its whole window: the edge padding of generators.py:217-221
            self.ring[fresh] = frame[fresh].unsqueeze(1)
            self.started |= fresh
        self.ring[:, self.head] = frame                      # overwrite the oldest slot
        self.head = (self.head + 1) % self.rf
        k = self.rf - self.head                              # unroll: oldest frame first, newest last
        self.window[:, :k] = self.ring[:, self.head:]
        self.window[:, k:] = self.ring[:, :self.head]
        with torch.no_grad():
            return self.model(self.window)[:, -1]
