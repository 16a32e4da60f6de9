"""Device-side counterpart of the reference's lib/track/sort.py (import as device.lib.track.sort): Sort(max_age,
min_hits).update(dets) with the Kalman filters, the assignment and the tracker list on the device
(gast_b200.tracking, DESIGN.md §8.8).  `from device.lib.track.sort import Sort` replaces `from track.sort import Sort`
(gen_kpts.py:34) with no other change.

Each update is one launch and one copy back.  Ids continue one process-wide count, KalmanBoxTracker.count, as the
reference's do across Sort instances.  dets must be float32 (person_boxes' and yolo_human_det's boxes are); only
their first four columns are read.  Where the reference raises (a NaN IoU, or a zero IoU denominator) this raises
GastError, as it does where the reference's arrays would go out of step (an infinite predicted box).
"""
import numpy as np
import torch

from gast_b200 import tracking as _T
from gast_b200.engine import GastError

__all__ = ['Sort', 'KalmanBoxTracker']


class KalmanBoxTracker:
    """holds the process-wide id count the reference keeps on its tracker class; the trackers live on the device"""
    count = 0


class Sort:
    def __init__(self, max_age=1, min_hits=3, capacity=256):
        self.max_age, self.min_hits = max_age, min_hits
        self._dev = _T.DeviceSort(1, max_age, min_hits, capacity)
        self._local_next = 0
        self._ids = np.empty(0, np.int64)      # this instance's tracker ids, in birth order, on the global count

    def update(self, dets=np.empty((0, 5), np.float32)):
        """Sort.update: dets (n, 4) or (n, 5) float32 -> (m, 5) float64 [x1, y1, x2, y2, id + 1]"""
        if isinstance(dets, torch.Tensor):
            dets = dets.cpu().numpy()
        dets = np.asarray(dets)
        if dets.size and dets.dtype != np.float32:
            raise GastError('Sort.update: dets must be float32, got %s' % dets.dtype)
        n = int(dets.shape[0]) if dets.ndim == 2 else 0
        if dets.size and (dets.ndim != 2 or dets.shape[1] < 4):
            raise GastError('Sort.update: dets (n, 4) or (n, 5) expected, got %s' % (dets.shape,))
        boxes = np.zeros((1, max(n, 1), 4), np.float32)
        if n:
            boxes[0, :n] = dets[:, :4]
        d = self._dev
        rows, counts, status = d.update_chunk(boxes, np.array([n], np.int32), skip_empty=False)
        cap = d.capacity
        packed = torch.cat([rows[0].reshape(-1).view(torch.uint8), counts.view(torch.uint8), status.view(torch.uint8),
                            d.state[:_T.HEADER_WORDS * 8]]).cpu().numpy()
        k = int(packed[cap * 40:cap * 40 + 4].view(np.int32)[0])
        st = int(packed[cap * 40 + 4:cap * 40 + 8].view(np.int32)[0])
        if st:
            raise GastError('Sort.update: %s' % _T.status_message(st))
        next_id = int(packed[cap * 40 + 8:].view(np.int64)[1])
        born = next_id - self._local_next
        if born:
            self._ids = np.concatenate([self._ids, KalmanBoxTracker.count + np.arange(born, dtype=np.int64)])
            KalmanBoxTracker.count += born
            self._local_next = next_id
        out = packed[:cap * 40].view(np.float64).reshape(cap, 5)[:k].copy()
        if k:
            out[:, 4] = self._ids[out[:, 4].astype(np.int64) - 1] + 1
        return out
