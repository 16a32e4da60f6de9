"""Frame-by-frame lifting of many concurrent keypoint streams (SURVEY.md §8f N4).

The reference's real-time model is a causal `SpatioTemporalModelOptimized1f` fed the last `receptive_field`
frames of one stream for every new frame (`gen_skes.py:43-69`, `tools/inference.py:19-110`): O(rf) work per
frame.  `PoseStream` produces the same poses with O(1) work per frame: the library keeps, per temporal stage, a
ring of that stage's past inputs for all streams (`csrc/stream.cuh`), so a pushed frame computes one new position per
layer.  A single-frame push of every stream runs the C ABI's `gast_stream_push_ex`; lockstep multi-frame and peek
calls go through the subset entries `gast_stream_push_subset` / `_peek_subset` on their null-table branch, and
calls on some of the streams or at unequal counts through the same entries with a table.  A stream's first frame
stands for its whole (edge-padded) history exactly like `UnchunkedGenerator` does (`common/generators.py:210-221`).

`PoseStream` takes causal and non-causal models.  A non-causal model returns the pose of frame t - pad when frame t
is pushed (`latency` = pad = (rf - 1) // 2; 0 for a causal model).  `end()` closes a stream's sequence: its next
`latency` pushes repeat the last frame (the generator's right padding) and return the remaining poses.  With
`augment=True` every push also runs the mirrored twin and averages it back, as every inference helper of the
reference does (`tools/inference.py:19-110`).  The poses of a sequence then equal
`UnchunkedGenerator([seq], pad, causal_shift, augment)` + `tools/inference.evaluate`.  Until then `peek()` returns
provisional poses of the pending frames, those of the sequence cut at its newest frame, without changing any stream.
`CausalStream` is the causal,
un-augmented restriction that returns the pose of the newest frame.  `export_streams` / `import_streams` move live
streams with their history into another pool of the same model (another size, eager or graphed), where they continue
as if they had never moved (`StreamSnapshot`, C ABI `gast_stream_export` / `gast_stream_import`).

The rings hold activations computed with the weights of the pushes that wrote them.  Any change to the model's
parameters or buffers (`load_state_dict`, an optimiser step, a training forward, which moves the BatchNorm running
statistics) therefore invalidates the history of every stream: the next push raises `GastError` unless `reset()`
(every stream) was called after the change.  Switching the GEMM core (`engine.set_gemm_core`) or the precision
between 'fp32' and 'tf32' (`engine.set_precision`, which the streams follow like every forward) changes no weight and
keeps the streams.  At 'fp16' the library keeps the rings in fp16 (half the bytes of history per stream), so a pool
records the ring type its state was allocated at: a switch to or from 'fp16' reallocates the state when every stream
is restarting and otherwise raises `GastError`.  A live pool changes precision by `export_streams` at the old
precision and `import_streams` into a new pool at the new one (snapshots are float32 at every precision).

`WindowStream` is the generic form for any callable network: a device ring of the last `rf` input frames and one
window forward per pushed frame (what the reference does; used for non-GAST callables and as the cross-check).
"""
import copy
import ctypes as C
import numpy as np
import torch

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
    the frame whose pose that push returns (-1 where nothing is due).  With `streams` (distinct indices), `advance`,
    `advance_many` and `peek` act on those streams only, in that order, as a book of those streams alone would."""

    def __init__(self, n, latency):
        self.n, self.latency = int(n), int(latency)
        self.fresh = np.ones(self.n, dtype=bool)            # the next push starts a new sequence
        self.length = np.zeros(self.n, dtype=np.int64)      # frames in the current sequence
        self.left = np.full(self.n, -1, dtype=np.int64)     # -1 live; k >= 0: k held pushes left (0 = idle)

    def _sel(self, streams):
        if streams is None:
            return slice(None)
        return np.asarray(streams, dtype=np.int64).reshape(-1)

    def check_streams(self, streams):
        """-> streams as an int64 array; ValueError unless they are 1 to n distinct indices in [0, n)"""
        s = np.asarray(streams).reshape(-1)
        if s.size and not np.issubdtype(s.dtype, np.integer):
            raise ValueError('streams must be integer stream indices (got %s)' % s.dtype)
        s = s.astype(np.int64)
        if s.size < 1 or (s < 0).any() or (s >= self.n).any() or np.unique(s).size != s.size:
            raise ValueError('streams must be 1 to %d distinct indices in [0, %d) (got %s)' % (self.n, self.n, s.tolist()))
        return s

    def _subset(self, streams, fn):
        """fn(book of the listed streams alone), then its state written back to those streams"""
        s = self.check_streams(streams)
        sub = copy.copy(self)
        sub.n, sub.fresh, sub.length, sub.left = s.size, self.fresh[s], self.length[s], self.left[s]
        out = fn(sub)
        self.fresh[s], self.length[s], self.left[s] = sub.fresh, sub.length, sub.left
        return out

    def rows(self, streams):
        """-> (fresh, length, left) of the listed streams, copies: their sequences, for `put_rows` of another book"""
        s = self.check_streams(streams)
        return self.fresh[s].copy(), self.length[s].copy(), self.left[s].copy()

    def put_rows(self, streams, rows):
        """the listed streams take the sequences `rows` (from `rows`): later calls treat them as the source book
        treated its streams (a fresh or idle stream stays so, an ending one keeps its pending poses)"""
        s = self.check_streams(streams)
        self.fresh[s], self.length[s], self.left[s] = rows

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

    def advance(self, streams=None):
        """-> (fresh, hold, index) of the next push; updates the state as that push does"""
        if streams is not None:
            return self._subset(streams, lambda b: b.advance())
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

    def advance_many(self, K, valid=None, streams=None):
        """-> (fresh (n,), hold (n, K), index (n, K)) of K consecutive pushes, as K calls of `advance()` return them,
        with `end([s])` before push valid[s] of every live stream s whose valid[s] < K (0 <= valid[s] <= K; None:
        no end).  Vectorised over the pushes: every stream is live up to its end and held from then on."""
        if streams is not None:
            return self._subset(streams, lambda b: b.advance_many(K, valid))
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

    def peek(self, K, streams=None):
        """-> index (n, K) of a peek of K pushes: what `advance_many(K)` returns after `end()` of every live stream,
        computed on a copy; this book is unchanged"""
        if streams is not None:
            return copy.deepcopy(self)._subset(streams, lambda b: b.peek(K))
        book = copy.deepcopy(self)
        book.end()
        return book.advance_many(K)[2]


class StreamSnapshot(object):
    """Some streams of a `PoseStream` moved out by `export_streams`, for `import_streams` into a pool of the same
    model (another n_streams, eager or graphed).

    data (m, copies, floats) float32: per stream its library snapshot (`gast_stream_export`: the input history and
    every ring in time order), copies = 2 with augment (the stream and its mirrored twin); fresh, length, left (m,):
    the streams' SequenceBook rows; counts (m,): their frame counts in the source pool.  The rest names what the
    history belongs to: arch (J, F, channels, filter widths, causal, latency), augment and the symmetry lists, the
    model object, the parameter signature of the weights that computed the history, and the device.  `to(device)`
    moves `data` only (e.g. to host memory and back); a snapshot is valid within the process that made it."""

    def __init__(self, data, fresh, length, left, counts, arch, augment, lists, model, sig, device):
        self.data, self.fresh, self.length, self.left, self.counts = data, fresh, length, left, counts
        self.arch, self.augment, self.lists, self.model, self.sig, self.device = arch, augment, lists, model, sig, device

    def to(self, device):
        c = copy.copy(self)
        c.data = self.data.to(device)
        return c


class PoseStream(object):
    """O(1)-per-frame lifting of `n_streams` concurrent streams with any non-dense model of the drop-in classes
    (`SpatioTemporalModel` or `SpatioTemporalModelOptimized1f`, causal or not: the weights are interchangeable).

    push(frame (n, J, F)) -> (poses (n, J, 3) CUDA, index (n,) CPU int64): poses[s] is the pose of frame index[s] of
    stream s's current sequence, or unspecified where index[s] == -1.  The kps/joints lists default to the
    reference's for J = 17 and J = 19; `augment=True` with another J needs all four.

    `push`, `push_frames` and `peek` take `streams`, a list of distinct stream indices: only those streams take part
    (their rows come in and go out in that order), the others sit the call out untouched.  Each stream then has its
    own frame count (`counts`); `step` is the smallest of them.  A `push` without `streams` while every count is
    equal runs the single-frame library entry gast_stream_push_ex at `step`.  Every other call runs the subset entries
    (gast_stream_push_subset / _peek_subset), whose cost follows the listed streams, not n_streams; a multi-frame or
    peek call without `streams` at equal counts lists every stream in order at `step`, which the library runs on the
    chunk path's plain lockstep addressing."""

    def __init__(self, model_pos, n_streams, augment=False, kps_left=None, kps_right=None, joints_left=None,
                 joints_right=None, device=None):
        from . import engine
        name = type(self).__name__
        if not hasattr(model_pos, '_gast_causal'):
            raise engine.GastError('%s needs a model of the drop-in classes (model/gast_net.py)' % name)
        if getattr(model_pos, '_gast_dense', False):
            raise engine.GastError('%s: the dense ablation has no streaming form' % name)
        engine.refuse_half(model_pos, name, 'streaming')
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
        self._delta = np.zeros(self.n, dtype=np.int64)   # counts - step (>= 0; all 0 while the streams are in step)
        self._sig = None                 # the handle's parameter signature at the last push
        self._state = None
        self._ring = None                # ring storage of the state: 'fp16' at the fp16 precision, else 'fp32'
        self._ws = None                  # library workspace of the largest call so far
        self._masks = None               # device [fresh | hold] masks of the largest push so far

    @property
    def counts(self):
        """(n,) int64: the frames pushed into each stream so far (held frames included)"""
        return self.step + self._delta

    def _select(self, streams):
        """-> None for a lockstep call, else the int64 stream indices of a subset call (every stream, in order, for
        streams=None once the counts differ)"""
        if streams is None:
            return np.arange(self.n, dtype=np.int64) if self._delta.any() else None
        return self._listed(streams)

    def _listed(self, streams):
        """-> streams as int64 indices; GastError unless they are 1 to n distinct indices in [0, n)"""
        try:
            return self.book.check_streams(streams)
        except ValueError as e:
            raise self.engine.GastError('%s: %s' % (type(self).__name__, e))

    def _set_counts(self, counts):
        """counts (n,) int64 become the streams' frame counts, with `step` kept at the smallest count"""
        self.step = int(counts.min())
        self._delta = counts - self.step

    def _advanced(self, sel, K):
        """the listed streams pushed K frames: counts[sel] += K"""
        counts = self.counts
        counts[sel] += K
        self._set_counts(counts)

    def _lib_streams(self, sel):
        """-> (copies, m) int64: the library streams of the pool streams sel (m,), the streams themselves and with
        augment their mirrored twins s + n.  Calls, their masks and the device counts list them copy-major (this
        array flattened); a snapshot's rows are stream-major (its transpose)."""
        return np.asarray(sel, dtype=np.int64)[None, :] + self.n * np.arange(self.copies)[:, None]

    def reset(self, streams=None):
        """Start new sequences on all (or the listed) streams with the next pushed frame; drop any pending tail."""
        self.book.reset(streams)

    def end(self, streams=None):
        """The current sequences of all (or the listed) streams ended with their last pushed frame.  Their next
        `latency` pushes ignore the caller's rows and return the remaining poses; then they are idle until reset."""
        self.book.end(streams)

    def _upload(self, fresh, hold):
        """-> device pointers of the fresh (m,) and hold (m, K) masks of a push, repeated for the mirrored half in the
        copy-major order of `_lib_streams` (None where no stream is set).  Every push reuses one buffer [fresh | hold]:
        the copy into it and the kernels that read it are ordered on the one stream the calls run on."""
        any_f, any_h = bool(fresh.any()), bool(hold.any())
        if not (any_f or any_h):
            return None, None
        mk = np.concatenate([np.tile(fresh.astype(np.int32), self.copies),
                             np.tile(hold.astype(np.int32), (self.copies, 1)).reshape(-1)])
        if self._masks is None or self._masks.numel() < mk.size:
            self._masks = torch.empty(mk.size, dtype=torch.int32, device=self.device)
        # pinned + non_blocking: no device sync; the caching host allocator keeps the buffer until the copy ran
        self._masks[:mk.size].copy_(torch.from_numpy(mk).pin_memory(), non_blocking=True)
        mm = self.copies * fresh.size
        return (self._masks.data_ptr() if any_f else None), (self._masks[mm:].data_ptr() if any_h else None)

    def _begin(self, h, st):
        """refresh the handle, refuse a push over history computed with other weights, allocate the state"""
        h.refresh(self.model, st)
        self._refuse_stale(self._sig, h.sig)
        self._alloc_state(h)

    def _refuse_stale(self, sig, now):
        """GastError unless a call may read the history that the weights of parameter signature `sig` computed (None:
        nothing pushed yet) when the weights are now those of `now`: the same weights, or every stream restarting"""
        if sig is not None and sig != now and not self.book.all_restarting():
            raise self.engine.GastError('%s: the model\'s parameters or buffers changed since the streams\' history '
                                        'was computed (load_state_dict, an optimiser step or a training forward) -- '
                                        'call reset() before pushing again' % type(self).__name__)

    def _alloc_state(self, h):
        """allocate the zeroed library state of the copies * n library streams on first use, after checking that the
        library's latency is the pool's; allocate it again at a precision with another ring storage type when every
        stream is restarting, else refuse (the history is stored in the old type)"""
        eng, lib = self.engine, h.lib
        ring = 'fp16' if eng.get_precision(self.model) == 'fp16' else 'fp32'
        if self._state is not None and ring != self._ring:
            if not self.book.all_restarting():
                raise eng.GastError("%s: the streams' history is stored in %s, the model is now set to precision %r, "
                                    "which keeps it in %s; set the precision back, or move the live streams with "
                                    "export_streams and import_streams into a pool used at the new precision"
                                    % (type(self).__name__, self._ring, eng.get_precision(self.model), ring))
            self._state = None
        if self._state is None:
            eng._check(lib.gast_stream_latency(h.h) != self.latency, 'gast_stream_latency')
            nb = eng._check_size(lib.gast_stream_state_bytes(h.h, self.copies * self.n), 'gast_stream_state_bytes')
            self._state = torch.zeros(nb, dtype=torch.uint8, device=self.device)
            self._ring = ring

    def _mirror(self, lib, x, x2, rows, st):
        """x2 (2, rows, J, F) = [x | x mirrored]: the library input of the twins of x (rows, J, F) (gast_tta_prepare)"""
        self.engine._check(lib.gast_tta_prepare(x.data_ptr(), x2.data_ptr(), rows, self.J, self.F, 0, 0,
                                                len(self.kps_left), self._kl, self._kr, st), 'gast_tta_prepare')

    def _merge(self, lib, y2, y, rows, st):
        """y (rows, J, 3) = the mean of the twins' poses y2 (2, rows, J, 3), the mirrored one un-mirrored
        (gast_tta_merge)"""
        self.engine._check(lib.gast_tta_merge(y2.data_ptr(), y.data_ptr(), rows, self.J, len(self.joints_left),
                                              self._jl, self._jr, st), 'gast_tta_merge')

    def push(self, frame, streams=None):
        """frame (n_streams, J, in_features): the newest 2D keypoints of every stream (normalised screen
        coordinates; rows of held streams are ignored) -> (poses (n, J, 3), index (n,) CPU int64).  With `streams`
        (m distinct indices): frame (m, J, F) -> (poses (m, J, 3), index (m,)) of those streams, in that order;
        the other streams are unchanged."""
        frame = torch.as_tensor(frame, dtype=torch.float32, device=self.device).contiguous()
        sel = self._select(streams)
        assert frame.shape == (self.n if sel is None else sel.size, self.J, self.F), frame.shape
        y, index = self._call(frame[:, None], 1, sel)
        return y[:, 0], index[:, 0]

    def push_frames(self, frames, valid=None, streams=None):
        """frames (n_streams, K, J, in_features): the next K frames of every stream -> (poses (n, K, J, 3) CUDA,
        index (n, K) CPU int64), what K calls of `push` with frames[:, k] return, in one library call
        (gast_stream_push_subset).  valid (n,) or None: only the first valid[s] frames of stream s belong to its
        sequence; a smaller value than K ends the sequence there (as `end([s])` before frame valid[s] would) and the
        rest of the chunk returns its tail.  Rows of held frames are ignored.  `reset()` / `end()` take effect at
        frame 0 of the call, as for `push`.  With `streams` (m distinct indices) frames, valid, poses and index have m
        rows, those streams' in that order, and only those streams advance.  A stream's flush is
        `push_frames(nan frames (1, latency, J, F), valid=[0], streams=[s])`."""
        frames = torch.as_tensor(frames, dtype=torch.float32, device=self.device).contiguous()
        sel = self._select(streams)
        assert frames.dim() == 4 and frames.shape[0] == (self.n if sel is None else sel.size) and \
            frames.shape[1] >= 1 and tuple(frames.shape[2:]) == (self.J, self.F), frames.shape
        return self._call(frames, int(frames.shape[1]), sel, valid)

    def peek(self, K=None, streams=None):
        """Provisional poses of the frames a non-causal model has not returned yet, without pushing -> (poses
        (n, K, J, 3) CUDA, index (n, K) CPU int64): what K more pushes would return if every stream's sequence ended
        at its newest frame (`end()` and K held pushes), in one library call (gast_stream_peek_subset).  Nothing
        changes: not the library state, not `step`, not the sequences.  Those poses are the reference's for the
        sequence cut at its newest frame (UnchunkedGenerator pads it with copies of that frame); the pushes still
        return the final poses `latency` pushes later.  K defaults to `latency`, 1 <= K <= latency.

        Lookahead: for a stream that pushed frames 0 .. l-1 of its sequence, row k is the pose of frame
        l - latency + k, so with K = latency the last row is the newest frame.  To show poses L frames behind the
        newest (0 <= L < latency), peek K = latency - L and take row K - 1: a smaller K costs less.  index[s, k] is
        the frame's position in stream s's sequence, -1 where nothing is due (ending streams with fewer poses left,
        idle or freshly reset streams, frames before the sequence's start); when no stream has a pose due the call
        launches nothing.  With `streams` (m distinct indices) poses and index have m rows, those streams' in that
        order, each stream peeked at its own frame count."""
        name = type(self).__name__
        if self.causal:
            raise self.engine.GastError('%s.peek needs a non-causal model: a causal model returns the pose of every '
                                        'pushed frame at once, so none is ever pending' % name)
        K = self.latency if K is None else int(K)
        if not 1 <= K <= self.latency:
            raise self.engine.GastError('%s.peek: K must be in [1, latency = %d] (got %d)' % (name, self.latency, K))
        return self._call(None, K, self._select(streams))

    def _call(self, frames, K, sel, valid=None):
        """The library call of a push of frames (m, K, J, F), or for frames None of a peek of K frames, over every
        stream (sel None: a lockstep call at `step`) or over the streams `sel`, each at its own count -> (poses
        (m, K, J, 3) CUDA, index (m, K) CPU int64).  A lockstep push of one frame without `valid` runs
        gast_stream_push_ex; every other call runs gast_stream_push_subset / _peek_subset, which run a lockstep call
        (every library stream listed in order at `step`) on the chunk path's own addressing.  A peek launches nothing
        when no pose is due, and leaves out the streams that never pushed a frame (their rows are unspecified)."""
        eng = self.engine
        if self.model.training:
            raise eng.GastError('%s: call .eval() on the model (streaming is inference)' % type(self).__name__)
        rows = np.arange(self.n, dtype=np.int64) if sel is None else sel
        y = torch.empty((rows.size, K, self.J, 3), dtype=torch.float32, device=self.device)
        if frames is None:
            index = self.book.peek(K, streams=sel)
            if not (index >= 0).any():
                self.last_launches = 0
                return y, torch.from_numpy(index)
            keep = self.counts[rows] >= 1
        else:
            keep = np.ones(rows.size, dtype=bool)
        single = sel is None and frames is not None and K == 1 and valid is None
        r = int(keep.sum())
        mm = self.copies * r
        h = eng.model_handle(self.model, self.device)
        lib = h.lib
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            self._begin(h, st)
            if single:
                fn, wb = 'gast_stream_workspace_bytes', lib.gast_stream_workspace_bytes(h.h, mm)
            else:
                fn, wb = 'gast_stream_subset_workspace_bytes', lib.gast_stream_subset_workspace_bytes(h.h, mm, K)
            wb = eng._check_size(wb, fn)
            if self._ws is None or self._ws.numel() < wb:
                self._ws = None
                self._ws = torch.empty(wb, dtype=torch.uint8, device=self.device)
            fresh_p = hold_p = None
            if frames is not None:
                fresh, hold, index = self.book.advance_many(K, valid, streams=sel)
                fresh_p, hold_p = self._upload(fresh, hold)
            yr = y if r == rows.size else torch.empty((r, K, self.J, 3), dtype=torch.float32, device=self.device)
            x, out = frames, yr
            if self.augment:
                if frames is not None:
                    # (2, m, K, J, F) = 2m library streams of K frames: [original | mirrored]
                    x = torch.empty((2,) + tuple(frames.shape), dtype=torch.float32, device=self.device)
                    self._mirror(lib, frames, x, r * K, st)
                out = torch.empty((2, r, K, self.J, 3), dtype=torch.float32, device=self.device)
            state = self._state.data_ptr()
            if single:
                fn, args = 'gast_stream_push_ex', (state, C.c_int64(self.step), x.data_ptr(), out.data_ptr(), mm,
                                                   fresh_p, hold_p)
            else:
                lib_streams = self._lib_streams(rows[keep]).reshape(-1).astype(np.int32)
                lib_steps = np.tile(self.counts[rows[keep]], self.copies).astype(np.int64)
                table = (state, self.copies * self.n, lib_streams.ctypes.data, lib_steps.ctypes.data, mm, K)
                if frames is None:
                    fn, args = 'gast_stream_peek_subset', table + (out.data_ptr(),)
                else:
                    fn, args = 'gast_stream_push_subset', table + (x.data_ptr(), out.data_ptr(), fresh_p, hold_p)
            eng._check(getattr(lib, fn)(h.h, *args, self._ws.data_ptr(), self._ws.numel(), st), fn)
            launches = int(lib.gast_last_launch_count(h.h))
            if self.augment:
                self._merge(lib, out, yr, r * K, st)
                launches += 2
            if r < rows.size:
                y[torch.from_numpy(np.flatnonzero(keep)).to(self.device)] = yr
        if frames is not None:
            self._sig = h.sig
            self._advanced(rows, K)
        self.last_launches = launches
        return y, torch.from_numpy(index)

    # ---- moving streams between pools -------------------------------------------------------------------------------
    def _arch(self):
        m = self.model
        return (self.J, self.F, int(m._gast_channels), tuple(int(w) for w in m.filter_widths), self.causal,
                self.latency)

    def _lists(self):
        return (self.kps_left, self.kps_right, self.joints_left, self.joints_right) if self.augment else None

    def _move_begin(self):
        """-> the refreshed handle, with the state allocated; refuses over history computed with other weights"""
        h = self.engine.model_handle(self.model, self.device)
        self._begin(h, torch.cuda.current_stream(self.device).cuda_stream)
        return h

    def _move(self, fn, h, sel, counts, data):
        """gast_stream_export / _import of data (m, copies, floats) for the streams sel at their counts: the library
        streams listed stream-major, so that the rows of data are (stream, copy)"""
        eng, lib = self.engine, h.lib
        lib_streams = self._lib_streams(sel).T.reshape(-1).astype(np.int32)
        lib_counts = np.repeat(np.asarray(counts, dtype=np.int64), self.copies)
        mm = lib_streams.size
        wb = eng._check_size(lib.gast_stream_move_workspace_bytes(h.h, mm), 'gast_stream_move_workspace_bytes')
        # not self._ws: a GraphedPoseStream's graph keeps that buffer's address
        ws = torch.empty(wb, dtype=torch.uint8, device=self.device)
        st = torch.cuda.current_stream(self.device).cuda_stream
        eng._check(getattr(lib, fn)(h.h, self._state.data_ptr(), self.copies * self.n, lib_streams.ctypes.data,
                                    lib_counts.ctypes.data, mm, data.data_ptr(), ws.data_ptr(), ws.numel(), st), fn)
        self.last_launches = int(lib.gast_last_launch_count(h.h))

    def export_streams(self, streams):
        """-> StreamSnapshot of the listed streams (distinct indices): their history on the device, their sequence
        bookkeeping and counts, for `import_streams` of a pool of the same model and architecture (any n_streams,
        eager or graphed).  Nothing changes in this pool.  Refused (GastError) like a push when the model's parameters
        or buffers changed since the last push and not every stream is restarting."""
        sel = self._listed(streams)
        with torch.cuda.device(self.device):
            h = self._move_begin()
            nf = self.engine._check_size(h.lib.gast_stream_snapshot_floats(h.h), 'gast_stream_snapshot_floats')
            data = torch.empty((sel.size, self.copies, nf), dtype=torch.float32, device=self.device)
            # a stream that never pushed is fresh or idle: its rows are never read, any count >= 1 will do
            self._move('gast_stream_export', h, sel, np.maximum(self.counts[sel], 1), data)
        return StreamSnapshot(data, *self.book.rows(sel), self.counts[sel].copy(), self._arch(), self.augment,
                              self._lists(), self.model, h.sig, self.device)

    def import_streams(self, snapshot, streams):
        """Overwrite the listed streams (distinct indices, one per exported stream, in the snapshot's order) with the
        exported streams: their history, their sequences (a fresh or idle stream stays so, an ending one keeps its
        pending poses) and the same poses from then on.  Each takes the count max(step, 1), the phase of this pool's
        lockstep calls.  The other streams are untouched.  Refused with GastError, changing nothing in either pool: a
        snapshot of another model object, architecture, `augment` or symmetry lists or device, a change of the
        model's parameters or buffers since the export (unless every exported stream is restarting), this pool's own
        weight-change rule, bad or duplicate streams, or a count that differs from the snapshot's."""
        eng, name = self.engine, type(self).__name__
        sel = self._listed(streams)
        if not isinstance(snapshot, StreamSnapshot):
            raise eng.GastError('%s.import_streams needs a StreamSnapshot from export_streams' % name)
        s = snapshot
        if sel.size != s.counts.size:
            raise eng.GastError('%s.import_streams: %d streams listed for a snapshot of %d' % (name, sel.size,
                                                                                              s.counts.size))
        if s.arch != self._arch() or s.augment != self.augment or s.lists != self._lists() or s.device != self.device:
            raise eng.GastError('%s.import_streams: the snapshot\'s architecture, augment, symmetry lists or device '
                                'differ from this pool\'s' % name)
        if s.model is not self.model:
            raise eng.GastError('%s.import_streams: the snapshot was exported from a pool of another model object'
                                % name)
        restarting = bool(np.all(s.fresh | (s.left == 0)))
        if not restarting and eng.param_sig(self.model) != s.sig:
            raise eng.GastError('%s.import_streams: the model\'s parameters or buffers changed since the export; the '
                                'exported history was computed with the old weights' % name)
        if tuple(s.data.shape[:2]) != (sel.size, self.copies):
            raise eng.GastError('%s.import_streams: snapshot data of shape %s' % (name, tuple(s.data.shape)))
        target = max(self.step, 1)
        with torch.cuda.device(self.device):
            h = self._move_begin()
            if s.data.shape[2] != h.lib.gast_stream_snapshot_floats(h.h):
                raise eng.GastError('%s.import_streams: snapshot data of shape %s' % (name, tuple(s.data.shape)))
            data = s.data.to(device=self.device, dtype=torch.float32).contiguous()
            self._move('gast_stream_import', h, sel, np.full(sel.size, target), data)
            self._moved_in(sel, target)
        self._sig = h.sig
        self.book.put_rows(sel, (s.fresh, s.length, s.left))
        counts = self.counts
        counts[sel] = target
        self._set_counts(counts)

    def _moved_in(self, sel, count):
        """device bookkeeping of streams imported at `count` (none here: the counts are the host's)"""


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

    def push(self, frame, streams=None):
        """frame (n_streams, J, in_features): the newest 2D keypoints of every stream (normalised screen
        coordinates).  Returns the 3D pose of that frame, (n_streams, J, 3).  With `streams` (m distinct indices):
        the frames and poses of those streams only, (m, J, F) -> (m, J, 3)."""
        return super(CausalStream, self).push(frame, streams=streams)[0]

    def push_frames(self, frames, streams=None):
        """frames (n_streams, K, J, in_features): the next K frames of every stream -> their 3D poses
        (n_streams, K, J, 3), what K calls of `push` return, in one library call.  `streams` as for `push`."""
        return super(CausalStream, self).push_frames(frames, streams=streams)[0]


class GraphedPoseStream(PoseStream):
    """`PoseStream` ticks replayed from one CUDA graph: a fixed pool of `n_streams` streams and K frames per stream.

    An eager push costs far more host time (Python bookkeeping and ~30-40 kernel launches) than device time at a
    few streams, and its time swings from call to call.  Here the launches of one tick,
    `[gast_tta_prepare] -> gast_stream_push_device -> [gast_stream_peek_device] -> [gast_tta_merge]`, are captured once
    over static buffers (input, poses, masks, the per-stream frame counts on the device, the state and the workspace)
    and replayed per tick; the library builds each stream's ring phase from the device counts, so the graph is right
    at every count.  The constructor takes `PoseStream`'s arguments plus K (frames per stream and tick) and `peek`: 0
    for none, else the tick also returns provisional poses of `peek` frames (1 <= peek <= latency), what
    `PoseStream.peek(peek)` returns right after the push.  The tick runs the chunk path, so it pays off for a few
    streams, most with a peek (one tick instead of two eager calls); hundreds of streams that all push every tick
    are faster with the eager lockstep push (DESIGN.md §8).

    push(frames (n, K, J, F), streams=None) -> (poses (n, K, J, 3), index (n, K) CPU int64) [+ (peek poses
    (n, peek, J, 3), peek index (n, peek))]: what `PoseStream.push_frames(frames[streams], streams=streams)` (and
    then `.peek(peek, streams=streams)`) returns, bit for bit, in the rows of the listed streams; the other streams sit
    the tick out unchanged, their rows of `frames` are not read and their index is -1.  The poses are views of static
    buffers that the next tick overwrites: copy them to keep them.  `reset()` / `end()` and `counts` are
    `PoseStream`'s; `counts` mirrors the device counts without any synchronisation.  `push_frames` and `peek` are
    refused: the ticks are the graph's.

    Refused with GastError before any replay: a model in training mode, an `engine.set_precision` or
    `engine.set_gemm_core` change since the capture, and a change of the model's parameters or buffers since the
    capture unless every stream is restarting (`PoseStream`'s rule after `reset()`), in which case the handle is
    refreshed and the tick captured again: a graph is never replayed over weights a later `gast_prepare` replaced."""

    def __init__(self, model_pos, n_streams, augment=False, kps_left=None, kps_right=None, joints_left=None,
                 joints_right=None, device=None, K=1, peek=0):
        super(GraphedPoseStream, self).__init__(model_pos, n_streams, augment=augment, kps_left=kps_left,
                                                kps_right=kps_right, joints_left=joints_left,
                                                joints_right=joints_right, device=device)
        name = type(self).__name__
        self.K, self.P = int(K), int(peek)
        if self.K < 1:
            raise self.engine.GastError('%s: K must be at least 1 (got %d)' % (name, self.K))
        if self.P and not 1 <= self.P <= self.latency:
            raise self.engine.GastError('%s: peek must be 0 or in [1, latency = %d] (got %d)'
                                        % (name, self.latency, self.P))
        n, N, J, dev = self.n, self.copies * self.n, self.J, self.device
        f32 = dict(dtype=torch.float32, device=dev)
        self._x = torch.zeros((n, self.K, J, self.F), **f32)
        self._y = torch.zeros((n, self.K, J, 3), **f32)
        self._py = torch.zeros((n, self.P, J, 3), **f32) if self.P else None
        # the library's [original | mirrored] twins of x, y and the peek poses
        self._x2 = torch.zeros((2, n, self.K, J, self.F), **f32) if self.augment else None
        self._y2 = torch.zeros((2, n, self.K, J, 3), **f32) if self.augment else None
        self._py2 = torch.zeros((2, n, self.P, J, 3), **f32) if self.augment and self.P else None
        # [fresh (N) | active (N) | hold (N, K)] on the device, and the pinned buffer every tick stages them in
        self._mask_dev = torch.zeros(N * (2 + self.K), dtype=torch.int32, device=dev)
        self._mask_host = torch.zeros(N * (2 + self.K), dtype=torch.int32).pin_memory()
        self._uploaded = torch.cuda.Event()     # recorded after the last copy out of _mask_host
        self._counts_dev = torch.zeros(N, dtype=torch.int64, device=dev)
        self.graph = None
        self._h = None
        self._mode = None                       # (GEMM core, precision) at the capture
        self._launches = 0

    def push_frames(self, frames, valid=None, streams=None):
        raise self.engine.GastError('%s: call push(); its ticks are replayed from the graph' % type(self).__name__)

    def peek(self, K=None, streams=None):
        raise self.engine.GastError('%s: construct it with peek=K; every tick then returns the peek'
                                    % type(self).__name__)

    def _mode_now(self):
        return (self.engine._FORCE_CORE['core'], self.engine.get_precision(self.model))

    def _tick(self, h, st):
        """enqueue one tick's library calls on stream `st` -> their launch count"""
        eng, lib = self.engine, h.lib
        n, N, K, P = self.n, self.copies * self.n, self.K, self.P
        ws, wn = self._ws.data_ptr(), self._ws.numel()
        fresh, active, hold = [t.data_ptr() for t in (self._mask_dev[:N], self._mask_dev[N:2 * N],
                                                      self._mask_dev[2 * N:])]
        state, counts = self._state.data_ptr(), self._counts_dev.data_ptr()
        x, y, py = self._x, self._y, self._py
        launches = 0
        if self.augment:
            self._mirror(lib, x, self._x2, n * K, st)
            x, y, py = self._x2, self._y2, self._py2
            launches += 1
        eng._check(lib.gast_stream_push_device(h.h, state, N, counts, active, K, x.data_ptr(), y.data_ptr(), fresh,
                                               hold, ws, wn, st), 'gast_stream_push_device')
        launches += int(lib.gast_last_launch_count(h.h))
        if self.augment:
            self._merge(lib, y, self._y, n * K, st)
            launches += 1
        if P:
            eng._check(lib.gast_stream_peek_device(h.h, state, N, counts, active, P, py.data_ptr(), ws, wn, st),
                       'gast_stream_peek_device')
            launches += int(lib.gast_last_launch_count(h.h))
            if self.augment:
                self._merge(lib, py, self._py, n * P, st)
                launches += 1
        return launches

    def _capture(self):
        """refresh the handle, size the state and the workspace, warm up outside capture, capture one tick"""
        eng = self.engine
        h = eng.model_handle(self.model, self.device)
        lib, N = h.lib, self.copies * self.n
        cur = torch.cuda.current_stream(self.device)
        side = torch.cuda.Stream(self.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            st = side.cuda_stream
            h.refresh(self.model, st)
            self._alloc_state(h)
            wb = max(eng._check_size(lib.gast_stream_device_workspace_bytes(h.h, N, k),
                                     'gast_stream_device_workspace_bytes') for k in (self.K, self.P) if k)
            if self._ws is None or self._ws.numel() < wb:
                self._ws = torch.empty(wb, dtype=torch.uint8, device=self.device)
            # warm-up (module loads, kernel attributes, the handle's lazy set-up): with every stream inactive it
            # changes no byte of the state and no count
            self._mask_dev[N:2 * N].zero_()
            self._tick(h, st)
        cur.wait_stream(side)
        self.graph = None
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            launches = self._tick(h, torch.cuda.current_stream(self.device).cuda_stream)
        self.graph, self._h, self._sig, self._mode, self._launches = graph, h, h.sig, self._mode_now(), launches

    def _ready(self):
        """refuse a tick over another GEMM core or precision, or over history computed with other weights; capture
        the tick when there is no graph yet, or again after a weight change with every stream restarting"""
        eng, name = self.engine, type(self).__name__
        if self.graph is not None:
            if self._mode_now() != self._mode:
                raise eng.GastError('%s: engine.set_precision or engine.set_gemm_core changed since the tick was '
                                    'captured; construct a new %s' % (name, name))
            now = eng.param_sig(self.model)
            if now != self._sig or self._h.sig != self._sig:   # new weights, or the handle prepared again
                self._refuse_stale(self._sig, now)
                self.graph = None
        if self.graph is None:
            self._capture()

    def _move_begin(self):
        self._ready()
        return self._h

    def _moved_in(self, sel, count):
        """the device counts of both library halves of the imported streams, ordered before the next replay on the
        current stream (the graph keeps the state and workspace addresses: no capture again)"""
        rows = self._lib_streams(sel).reshape(-1)
        self._counts_dev[torch.from_numpy(rows).to(self.device)] = int(count)

    def push(self, frames, streams=None):
        eng, name = self.engine, type(self).__name__
        if self.model.training:
            raise eng.GastError('%s: call .eval() on the model (streaming is inference)' % name)
        sel = np.arange(self.n, dtype=np.int64) if streams is None else self._select(streams)
        frames = torch.as_tensor(frames, dtype=torch.float32)
        assert tuple(frames.shape) == tuple(self._x.shape), frames.shape
        with torch.cuda.device(self.device):
            self._ready()
            n, N, K, P = self.n, self.copies * self.n, self.K, self.P
            fresh, hold, index = self.book.advance_many(K, streams=sel)
            idx = np.full((n, K), -1, dtype=np.int64)
            idx[sel] = index
            ls = self._lib_streams(sel)
            mk = self._mask_host.numpy()
            self._uploaded.synchronize()                       # the previous tick's copy has left the buffer
            mk[:] = 0
            mk[ls[:, fresh]] = 1
            mk[N + ls] = 1
            mk[2 * N:].reshape(N, K)[ls] = hold
            self._mask_dev.copy_(self._mask_host, non_blocking=True)
            self._uploaded.record()
            self._x.copy_(frames, non_blocking=True)
            self.graph.replay()
        self._advanced(sel, K)
        self.last_launches = self._launches
        out = (self._y, torch.from_numpy(idx))
        if P:
            pidx = np.full((n, P), -1, dtype=np.int64)
            pidx[sel] = self.book.peek(P, streams=sel)
            out += (self._py, torch.from_numpy(pidx))
        return out


def lift_sequences(model_pos, sequences, n_streams=64, chunk=256, augment=False, kps_left=None, kps_right=None,
                   joints_left=None, joints_right=None):
    """Whole-sequence lifting in bounded memory: sequences [(T_i, J, in_features)] -> [(T_i, J, 3) CUDA tensors],
    the poses `UnchunkedGenerator` + the model forward (+ the TTA merge with `augment=True`) compute for each
    sequence, i.e. what `tta.evaluate_sequence` returns.  The sequences are packed onto `n_streams` streams of a
    `PoseStream` and pushed `chunk` frames at a time; a stream starts its next sequence at the first chunk after the
    last pose of its previous one.  The library's scratch memory depends on (n_streams, chunk), not on T_i."""
    from . import engine
    engine.refuse_half(model_pos, 'lift_sequences', 'streaming')
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
