"""SORT (lib/track/sort.py) on the device: the Kalman box trackers, the IoU association and the tracker list's life
cycle for a chunk of frames of one or many videos in one launch (csrc/track.cuh, DESIGN.md §8.8).

`DeviceSort(sequences, max_age, min_hits, capacity, first_id)` holds S independent Sort states on the device.
`update_chunk(boxes, counts)` takes person_boxes' outputs for K frames ((K, max_det, 4) float32 and (K,) int32, or
(S, K, max_det, 4) and (S, K) for S sequences) and returns the reference's per-frame update() rows, their counts and
each sequence's status word as CUDA tensors without waiting for the device.  `host_tracks` makes one copy and returns
video_boxes' list: a (k, 5) float64 array [x1, y1, x2, y2, id + 1] per frame, None for a skipped frame.

Counts, ids and row order equal the reference's; the boxes are fp64 within a few ulps of it (S^-1 and the products
with the Kalman gain cannot follow OpenBLAS's order).  Where the reference raises (a NaN IoU or a zero IoU
denominator) or goes out of step (an infinite predicted box), and where a count or the tracker list does not fit,
the sequence's status word is set and host_tracks raises GastError.
"""
import numpy as np
import torch

from . import _lib as L
from .engine import GastError, _launch, _p
from .keypoints2d import _device, _on_device

SKIP_EMPTY = 1                   # GAST_SORT_SKIP_EMPTY
STATUS = {1: 'a frame has more detections than max_det', 2: 'the tracker list outgrew its capacity',
          4: 'an IoU the reference refuses (NaN, or a zero denominator)',
          8: 'a predicted box with an infinite coordinate', 16: 'a state not initialised for this capacity'}
HEADER_WORDS = 8                 # int64: frame_count, next id, trackers, status, max_age, min_hits, capacity, tag


def status_message(word):
    return '; '.join(m for b, m in STATUS.items() if int(word) & b) or 'status %d' % int(word)


class DeviceSort:
    """Sort(max_age, min_hits) for `sequences` videos at once, its state on the device.  Ids start at first_id (an
    int, or one per sequence), as KalmanBoxTracker.count would have them; capacity bounds each tracker list."""

    def __init__(self, sequences=1, max_age=1, min_hits=3, capacity=256, first_id=0, device=None):
        self.S, self.capacity = int(sequences), int(capacity)
        self.max_age, self.min_hits = int(max_age), int(min_hits)
        if self.S < 1 or self.max_age < 0 or self.min_hits < 0:
            raise GastError('tracking: sequences >= 1, max_age >= 0 and min_hits >= 0 expected')
        lib = L.load()
        n = lib.gast_sort_state_bytes(self.S, self.capacity)
        if n == 0:
            raise GastError('tracking: %s' % L.last_error())
        self.device = _device(device)
        self.state_bytes = int(n) // self.S
        self.state = torch.empty(int(n), dtype=torch.uint8, device=self.device)
        ids = np.broadcast_to(np.asarray(first_id, np.int64), (self.S,))
        first = _on_device(ids, torch.int64, self.device, 'first_id')
        _launch(self.device, 'gast_sort_init', _p(self.state), self.S, self.capacity, self.max_age, self.min_hits,
                _p(first))

    def header(self):
        """(S, 8) int64 view of each sequence's header words on the device (index 1: the next id)"""
        return self.state.view(self.S, self.state_bytes)[:, :HEADER_WORDS * 8].contiguous().view(torch.int64)

    def update_chunk(self, boxes, counts, skip_empty=True):
        """Sort.update for each of K frames in order.  boxes (K, max_det, 4) / (S, K, max_det, 4) float32, counts
        (K,) / (S, K) int32, numpy or CUDA.  Returns rows ((S,) K, capacity, 5) float64 (rows past the count are not
        written), counts ((S,) K) int32 (-1: a frame skipped because it has no box or only zero boxes) and status
        (S,) int32, all on the device; nothing waits for the device."""
        if isinstance(boxes, torch.Tensor):
            if boxes.dtype != torch.float32:
                raise GastError('tracking: boxes must be float32, got %s' % boxes.dtype)
        elif np.asarray(boxes).dtype != np.float32:
            raise GastError('tracking: boxes must be float32, got %s' % np.asarray(boxes).dtype)
        shape = tuple(boxes.shape)
        single = len(shape) == 3
        if single:
            shape = (1,) + shape
        if len(shape) != 4 or shape[-1] != 4 or shape[0] != self.S:
            raise GastError('tracking: boxes (K, max_det, 4) or (%d, K, max_det, 4) expected, got %s'
                            % (self.S, tuple(boxes.shape)))
        S, K, M = shape[0], shape[1], shape[2]
        if isinstance(counts, torch.Tensor):
            if counts.dtype not in (torch.int32, torch.int64):
                raise GastError('tracking: counts must be integers, got %s' % counts.dtype)
        elif not np.issubdtype(np.asarray(counts).dtype, np.integer):
            raise GastError('tracking: counts must be integers, got %s' % np.asarray(counts).dtype)
        if tuple(counts.shape) != ((K,) if single else (S, K)):
            raise GastError('tracking: counts %s for boxes %s' % (tuple(counts.shape), tuple(boxes.shape)))
        dev = self.device
        b = _on_device(boxes, torch.float32, dev, 'boxes')
        n = _on_device(counts, torch.int32, dev, 'counts')
        rows = torch.empty((S, K, self.capacity, 5), dtype=torch.float64, device=dev)
        out_counts = torch.empty((S, K), dtype=torch.int32, device=dev)
        status = torch.empty(S, dtype=torch.int32, device=dev)
        _launch(dev, 'gast_sort_update', _p(self.state), S, self.capacity, K, _p(b), _p(n), M,
                SKIP_EMPTY if skip_empty else 0, _p(rows), _p(out_counts), _p(status))
        if single:
            return rows[0], out_counts[0], status
        return rows, out_counts, status


def host_tracks(rows, counts, status):
    """update_chunk's outputs -> the per-frame list video_boxes returns ((k, 5) float64 per frame, None for a skipped
    frame), or one such list per sequence for (S, K, ...) outputs.  One copy to the host; GastError when a status
    word is set."""
    single = rows.dim() == 3
    R = rows[None] if single else rows
    N = counts[None] if single else counts
    S, K, cap = int(R.shape[0]), int(R.shape[1]), int(R.shape[2])
    packed = torch.cat([R.reshape(-1).view(torch.uint8), N.reshape(-1).view(torch.uint8),
                        status.reshape(-1).view(torch.uint8)]).cpu().numpy()
    nr = S * K * cap * 5 * 8
    r = packed[:nr].view(np.float64).reshape(S, K, cap, 5)
    n = packed[nr:nr + S * K * 4].view(np.int32).reshape(S, K)
    st = packed[nr + S * K * 4:].view(np.int32)
    if st.any():
        bad = int(np.flatnonzero(st)[0])
        raise GastError('tracking: sequence %d: %s' % (bad, status_message(st[bad])))
    out = [[None if n[s, t] < 0 else r[s, t, :n[s, t]].copy() for t in range(K)] for s in range(S)]
    return out[0] if single else out
