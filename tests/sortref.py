"""A numpy restatement of SORT as the reference runs it (lib/track/sort.py with numba's iou, scipy 1.18's
linear_sum_assignment and filterpy 1.4.5's KalmanFilter), and the integer formulas of the tests' detections.

- `lsap` restates scipy's rectangular_lsap.cpp (the shortest augmenting path solver) in pure Python: the transpose
  of a tall matrix, the fp64 cost, the `remaining` list with swap-removal, the tie rule (a strictly lower reduced cost,
  or an equal one at an unassigned column) and the output sorted by row.
- `iou` restates the numba function: the detection's area in float32, everything else fp64, ZeroDivisionError on a
  zero denominator as numba's Python error model raises it.
- `KalmanFilter` is filterpy 1.4.5's filter reduced to what SORT calls, with its defaults and equations (not checked
  against filterpy itself, which is not installed here); tests/golden/make_golden_sort.py hands it to the unmodified
  reference as `filterpy.kalman.KalmanFilter`.
- `Sort` is the reference's tracker restated on those three with the same numpy calls, so it equals the goldens bit
  for bit.  DESIGN.md §8.8 writes the formulas down.
"""
import numpy as np

IOU_THRESHOLD = np.float32(0.3)


# ---------------------------------------------------------------------------------------------- assignment
def lsap(cost):
    """scipy.optimize.linear_sum_assignment(cost) (minimise) -> (rows, cols) int64 arrays, sorted by row"""
    c = np.asarray(cost, dtype=np.float64)
    if c.ndim != 2:
        raise ValueError('expected a matrix')
    nr, nc = c.shape
    if nr == 0 or nc == 0:
        return np.empty(0, np.int64), np.empty(0, np.int64)
    tr = nc < nr
    if tr:
        c = c.T
        nr, nc = nc, nr
    if np.isnan(c).any() or (c == -np.inf).any():
        raise ValueError('matrix contains invalid numeric entries')
    cost = c.ravel().tolist()
    u = [0.0] * nr
    v = [0.0] * nc
    path = [-1] * nc
    col4row = [-1] * nr
    row4col = [-1] * nc
    for cur in range(nr):
        spc = [np.inf] * nc
        SR = [False] * nr
        SC = [False] * nc
        remaining = [nc - it - 1 for it in range(nc)]
        num_remaining = nc
        min_val = 0.0
        i = cur
        sink = -1
        while sink == -1:
            index = -1
            lowest = np.inf
            SR[i] = True
            base = i * nc
            for it in range(num_remaining):
                j = remaining[it]
                r = min_val + cost[base + j] - u[i] - v[j]
                if r < spc[j]:
                    path[j] = i
                    spc[j] = r
                if spc[j] < lowest or (spc[j] == lowest and row4col[j] == -1):
                    lowest = spc[j]
                    index = it
            min_val = lowest
            if min_val == np.inf:
                raise ValueError('cost matrix is infeasible')
            j = remaining[index]
            if row4col[j] == -1:
                sink = j
            else:
                i = row4col[j]
            SC[j] = True
            num_remaining -= 1
            remaining[index] = remaining[num_remaining]
        u[cur] += min_val
        for r in range(nr):
            if SR[r] and r != cur:
                u[r] += min_val - spc[col4row[r]]
        for j in range(nc):
            if SC[j]:
                v[j] -= min_val - spc[j]
        j = sink
        while True:
            r = path[j]
            row4col[j] = r
            col4row[r], j = j, col4row[r]
            if r == cur:
                break
    if tr:
        order = sorted(range(nr), key=lambda k: col4row[k])
        return np.array([col4row[k] for k in order], np.int64), np.array(order, np.int64)
    return np.arange(nr, dtype=np.int64), np.array(col4row, np.int64)


# ---------------------------------------------------------------------------------------------- the tracker
def iou(det, trk):
    """numba's iou(det, trk): det a float32 row, trk a float64 row; the result is stored as float32"""
    xx1 = np.maximum(det[0], trk[0])
    yy1 = np.maximum(det[1], trk[1])
    xx2 = np.minimum(det[2], trk[2])
    yy2 = np.minimum(det[3], trk[3])
    wh = np.maximum(0., xx2 - xx1) * np.maximum(0., yy2 - yy1)
    area_det = (det[2] - det[0]) * (det[3] - det[1])               # float32
    den = np.float64(area_det) + (trk[2] - trk[0]) * (trk[3] - trk[1]) - wh
    if den == 0:
        raise ZeroDivisionError('division by zero')
    return np.float32(wh / den)


def bbox_to_z(b):
    """float32 in, float32 out: NumPy 2 keeps w / float(h) in float32"""
    w = b[2] - b[0]
    h = b[3] - b[1]
    return np.array([b[0] + w / 2., b[1] + h / 2., w * h, w / float(h)]).reshape((4, 1))


def x_to_bbox(x):
    w = np.sqrt(x[2] * x[3])
    h = x[2] / w
    return np.array([x[0] - w / 2., x[1] - h / 2., x[0] + w / 2., x[1] + h / 2.]).reshape((1, 4))


class KalmanFilter:
    """filterpy 1.4.5's KalmanFilter as SORT drives it: defaults x = 0, P = Q = F = I, H = 0, R = I; predict
    x = Fx, P = alpha^2 F P F' + Q; update y = z - Hx, S = H P H' + R, K = P H' inv(S), x = x + Ky and the Joseph form
    P = (I - KH) P (I - KH)' + K R K'"""

    def __init__(self, dim_x, dim_z, dim_u=0):
        self.dim_x, self.dim_z, self.dim_u = dim_x, dim_z, dim_u
        self.x = np.zeros((dim_x, 1))
        self.P = np.eye(dim_x)
        self.Q = np.eye(dim_x)
        self.B = None
        self.F = np.eye(dim_x)
        self.H = np.zeros((dim_z, dim_x))
        self.R = np.eye(dim_z)
        self._alpha_sq = 1.
        self._I = np.eye(dim_x)
        self.inv = np.linalg.inv

    def predict(self, u=None, B=None, F=None, Q=None):
        F = self.F if F is None else F
        Q = self.Q if Q is None else (np.eye(self.dim_x) * Q if np.isscalar(Q) else Q)
        B = self.B if B is None else B
        if B is not None and u is not None:
            self.x = np.dot(F, self.x) + np.dot(B, u)
        else:
            self.x = np.dot(F, self.x)
        self.P = self._alpha_sq * np.dot(np.dot(F, self.P), F.T) + Q

    def update(self, z, R=None, H=None):
        R = self.R if R is None else (np.eye(self.dim_z) * R if np.isscalar(R) else R)
        H = self.H if H is None else H
        z = np.atleast_2d(z)
        if z.shape[1] == self.dim_z:
            z = z.T
        self.y = z - np.dot(H, self.x)
        PHT = np.dot(self.P, H.T)
        self.S = np.dot(H, PHT) + R
        self.SI = self.inv(self.S)
        self.K = np.dot(PHT, self.SI)
        self.x = self.x + np.dot(self.K, self.y)
        I_KH = self._I - np.dot(self.K, H)
        self.P = np.dot(np.dot(I_KH, self.P), I_KH.T) + np.dot(np.dot(self.K, R), self.K.T)


F_SORT = np.array([[1, 0, 0, 0, 1, 0, 0], [0, 1, 0, 0, 0, 1, 0], [0, 0, 1, 0, 0, 0, 1], [0, 0, 0, 1, 0, 0, 0],
                   [0, 0, 0, 0, 1, 0, 0], [0, 0, 0, 0, 0, 1, 0], [0, 0, 0, 0, 0, 0, 1]])
H_SORT = np.array([[1, 0, 0, 0, 0, 0, 0], [0, 1, 0, 0, 0, 0, 0], [0, 0, 1, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0, 0]])


class Track:
    """one KalmanBoxTracker: SORT's constant-velocity box filter and its counters"""

    def __init__(self, box, tid):
        kf = KalmanFilter(dim_x=7, dim_z=4)
        kf.F, kf.H = F_SORT, H_SORT
        kf.R[2:, 2:] *= 10.
        kf.P[4:, 4:] *= 1000.
        kf.P *= 10.
        kf.Q[-1, -1] *= 0.01
        kf.Q[4:, 4:] *= 0.01
        kf.x[:4] = bbox_to_z(box)
        self.kf, self.id = kf, tid
        self.time_since_update = self.hits = self.hit_streak = self.age = 0

    def predict(self):
        if self.kf.x[6] + self.kf.x[2] <= 0:
            self.kf.x[6] *= 0.0
        self.kf.predict()
        self.age += 1
        if self.time_since_update > 0:
            self.hit_streak = 0
        self.time_since_update += 1
        return x_to_bbox(self.kf.x)[0]

    def update(self, box):
        self.time_since_update = 0
        self.hits += 1
        self.hit_streak += 1
        self.kf.update(bbox_to_z(box))


def associate(dets, trks):
    """(matches (k, 2), unmatched detections, unmatched trackers) in the reference's orders"""
    if len(trks) == 0:
        return np.empty((0, 2), int), list(range(len(dets))), []
    m = np.zeros((len(dets), len(trks)), np.float32)
    for d in range(len(dets)):
        for t in range(len(trks)):
            m[d, t] = iou(dets[d], trks[t])
    rows, cols = lsap(-m)
    um_d = [d for d in range(len(dets)) if d not in rows]
    um_t = [t for t in range(len(trks)) if t not in cols]
    matches = []
    for d, t in zip(rows, cols):
        if m[d, t] < IOU_THRESHOLD:
            um_d.append(int(d))
            um_t.append(int(t))
        else:
            matches.append((int(d), int(t)))
    return np.array(matches, int).reshape(-1, 2), um_d, um_t


class Sort:
    """the reference's Sort(max_age, min_hits); ids start at first_id (KalmanBoxTracker.count), and `next_id` is where
    the count stands"""

    def __init__(self, max_age=1, min_hits=3, first_id=0):
        self.max_age, self.min_hits = max_age, min_hits
        self.trackers = []
        self.frame_count = 0
        self.next_id = first_id

    def update(self, dets):
        self.frame_count += 1
        trks = np.zeros((len(self.trackers), 5))
        nan_rows = []
        for t, trk in enumerate(self.trackers):
            pos = trk.predict()
            trks[t, :4] = pos
            if np.any(np.isnan(pos)):
                nan_rows.append(t)
        finite = np.all(np.isfinite(trks), axis=1)
        if any(not finite[t] for t in range(len(trks)) if t not in nan_rows):
            raise IndexError('an infinite predicted box: trks and trackers out of step')
        trks = trks[finite]
        for t in reversed(nan_rows):
            self.trackers.pop(t)
        matches, um_d, um_t = associate(dets, trks)
        for t, trk in enumerate(self.trackers):
            if t not in um_t:
                trk.update(dets[matches[matches[:, 1] == t][0, 0], :])
        for d in um_d:
            self.trackers.append(Track(dets[d, :], self.next_id))
            self.next_id += 1
        out = []
        for i in range(len(self.trackers) - 1, -1, -1):
            trk = self.trackers[i]
            if trk.time_since_update < 1 and (trk.hit_streak >= self.min_hits or self.frame_count <= self.min_hits):
                out.append(np.concatenate((x_to_bbox(trk.kf.x)[0], [trk.id + 1])))
            if trk.time_since_update > self.max_age:
                self.trackers.pop(i)
        return np.array(out).reshape(-1, 5)


# ---------------------------------------------------------------------------------------------- detections
def _boxes(rows, cols=4):
    """integer hundredths (x1, y1, x2, y2[, score]) -> float32 boxes, as person_boxes' round(v, 2) leaves them"""
    a = np.asarray(rows, np.float64).reshape(-1, cols) / 100
    return a.astype(np.float32)


def _person(t, x0, y0, vx, vy, w=18000, h=42000):
    x = x0 + vx * t + (7 * t) % 23
    y = y0 + vy * t + (5 * t) % 17
    return [x, y, x + w + (3 * t) % 29, y + h + (11 * t) % 31]


def scenarios():
    """name -> (max_age, min_hits, [per-frame float32 detections]) for the goldens"""
    S = {}
    S['baseball'] = (1, 3, [_boxes([_person(t, 60000, 30000, 150, 40)]) for t in range(277)])
    S['crossing'] = (1, 3, [_boxes([_person(t, 20000, 30000, 1500, 0), _person(t, 110000, 31000, -1500, 0)])
                            for t in range(60)])
    frames = []
    for t in range(80):
        rows = [_person(t, 10000, 20000, 300, 0)]
        if 10 <= t < 40:
            rows.append(_person(t, 90000, 25000, -200, 50, 15000, 38000))
        if 25 <= t < 70:
            rows.append(_person(t, 50000, 60000, 0, -300, 16000, 35000))
        frames.append(_boxes(rows))
    S['births_deaths'] = (1, 3, frames)
    frames = []
    for t in range(40):
        rows = [_person(t, 30000, 20000, 200, 100)]
        if t not in (10, 20, 21):                     # gone for 1 frame, then for 2
            rows.append(_person(t, 120000, 20000, -100, 0))
        frames.append(_boxes(rows))
    S['missing'] = (1, 3, frames)
    S['missing_age3'] = (3, 2, frames)
    S['warmup'] = (1, 3, [_boxes([_person(t, 10000 + 40000 * k, 20000, 100, 0) for k in range(min(t + 1, 4))])
                          for t in range(8)])
    frames = []
    for t in range(30):
        rows = [_person(t, 20000, 20000, 100, 0)]
        if t % 3:
            rows += [[150000 + 3000 * k, 5000 + 4000 * k, 152000 + 3000 * k, 8000 + 4000 * k]
                     for k in range(2 + t % 4)]     # small far boxes: every IoU with the tracked person is 0
        frames.append(_boxes(rows))
    S['zero_ties'] = (1, 1, frames)
    S['many_ties'] = (2, 0, [_boxes([[1000 * ((k * 7 + t) % 19), 1000 * ((k * 5 + 3 * t) % 13),
                                      1000 * ((k * 7 + t) % 19) + 800, 1000 * ((k * 5 + 3 * t) % 13) + 900]
                                     for k in range(1 + (t * 5) % 9)]) for t in range(40)])
    frames = []
    for t in range(30):
        w = max(40000 - 3000 * t * t // 4, 100)     # shrinks fast, then holds
        frames.append(_boxes([[50000, 50000, 50000 + w, 50000 + 2 * w]]))
    S['shrink'] = (1, 3, frames)
    S['five_col'] = (1, 3, [_boxes([_person(t, 20000, 30000, 200, 0) + [90 - t], _person(t, 90000, 30000, -200, 0)
                                    + [80 + t]], 5) for t in range(25)])
    # an inverted box whose float32 area cancels the tracked box's: the IoU's denominator is 0 and numba raises
    S['zero_den'] = (1, 3, [_boxes([[10000, 10000, 15000, 20000]]), _boxes([[10000, 10000, 15000, 20000]]),
                            _boxes([[15000, 10000, 10000, 20000]])])
    # a NaN coordinate: linear_sum_assignment refuses the NaN IoU
    nan = _boxes([[10000, 10000, 15000, 20000]])
    nan_frame = nan.copy()
    nan_frame[0, 2] = np.nan
    S['nan_box'] = (1, 3, [nan, nan, nan_frame])
    return S


def random_sequence(T, seed, max_persons=12, alive=0.5):
    """T frames of 0 .. max_persons walking persons (each present at the start with probability `alive`) with clutter
    boxes and dropouts, float32 in hundredths"""
    rng = np.random.default_rng(seed)
    P = max_persons
    pos = rng.integers(0, 150000, size=(P, 2)).astype(np.int64)
    vel = rng.integers(-400, 401, size=(P, 2))
    size = np.stack([rng.integers(4000, 30000, P), rng.integers(8000, 60000, P)], 1)
    alive = rng.random(P) < alive
    frames = []
    for t in range(T):
        flip = rng.random(P) < 0.01
        alive = alive ^ flip
        pos += vel
        bounce = (pos < 0) | (pos > 170000)
        vel[bounce] *= -1
        pos = np.clip(pos, 0, 170000)
        rows = []
        for p in range(P):
            if alive[p] and rng.random() > 0.05:                   # dropouts
                j = rng.integers(-300, 301, 4)
                x1, y1 = pos[p] + j[:2]
                rows.append([x1, y1, x1 + size[p, 0] + j[2], y1 + size[p, 1] + j[3]])
        for _ in range(rng.poisson(0.4)):                          # clutter
            x1, y1 = rng.integers(0, 180000, 2)
            rows.append([x1, y1, x1 + rng.integers(500, 9000), y1 + rng.integers(500, 9000)])
        order = rng.permutation(len(rows))
        frames.append(_boxes([rows[k] for k in order]))
    return frames


def run(frames, max_age=1, min_hits=3, first_id=0, skip_empty=False):
    """the restatement over frames; a skipped frame (skip_empty and no box or all zero) gives None"""
    s = Sort(max_age, min_hits, first_id)
    out = []
    for d in frames:
        if skip_empty and (len(d) == 0 or not d.any()):
            out.append(None)
        else:
            out.append(s.update(d))
    return out


def pack(frames, max_det=None):
    """per-frame detections -> (K, max_det, 4) float32 boxes (zero past the count) and (K,) int32 counts"""
    K = len(frames)
    n = np.array([len(d) for d in frames], np.int32)
    M = int(max_det if max_det is not None else max(1, n.max() if K else 1))
    boxes = np.zeros((K, M, 4), np.float32)
    for t, d in enumerate(frames):
        boxes[t, :min(len(d), M)] = d[:M, :4]
    return boxes, n
