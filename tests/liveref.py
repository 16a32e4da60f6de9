"""numpy restatement of csrc/live.cuh, the live tick's own steps (gen_img_kpts -> the causal streams ->
revise_skes_real_time), vectorised over slots:
  select / slot_geometry   gast_live_slots' track selection (gen_img_kpts:146-150, no round(v, 2)) and box geometry;
  SlotBook                 its slot rule: ids keep their slots, new ids take free slots, then the slots seen longest
                           ago, and a slot whose id changes restarts its stream;
  inputs                   gast_live_inputs: h36m_coco_format, keep and valid of one frame, revise_kpts' repair and
                           normalize_screen_coordinates;
  place                    gast_live_place: revise_skes_real_time over a camera's active slots, zeros elsewhere.
numpy's float32 / float64 element-wise operations round to nearest and are never fused, as the kernels' intrinsics."""
import numpy as np

import recordsref as R
from oracle.pipeline_oracle import F32, _COCO_TO_H36M, coco_h36m

ST_TRACKS, ST_NONFINITE, ST_EMPTY, ST_MATRIX = R.ST_TRACKS, R.ST_NONFINITE, R.ST_EMPTY, R.ST_MATRIX
ROT = np.array([0.14070565, -0.15007018, -0.7552408, 0.62232804], dtype=np.float32)


def select(k, num_person, cap):
    """the row indices gen_img_kpts keeps of a frame of k tracks, in selection order, and its status bit"""
    n = R.rec_count(k, num_person, cap)
    if n < 0:
        return [], ST_TRACKS
    return ([0] if k == 1 else [k - 1 - p for p in range(n)]), 0


def slot_geometry(boxes, H, W, image_size, heatmap_size):
    """unrounded boxes (n, 4) float64 -> centers, scales (n, 2) float32, forward and inverse (n, 2, 3) float64 and the
    status bits (n,); a box with a bit is inactive: zero center, scale and matrices"""
    b = np.asarray(boxes, np.float64).reshape(-1, 4)
    c, s, fwd, inv, bits = R.box_matrices(b, H, W, image_size, heatmap_size)
    with np.errstate(invalid='ignore'):
        bits = bits | np.where(np.isfinite(fwd.reshape(-1, 6)).all(1), 0, ST_MATRIX)
    bad = bits != 0
    c[bad], s[bad], fwd[bad], inv[bad] = 0, 0, 0, 0
    return c, s, fwd, inv, bits


class SlotBook(object):
    """one camera's slots: id (-1 none), last tick selected (-1 never), restart flag"""

    def __init__(self, P):
        self.P = P
        self.ids = np.full(P, -1, np.int64)
        self.seen = np.full(P, -1, np.int64)
        self.fresh = np.ones(P, bool)

    def assign(self, ids, tick):
        """the selected ids (in selection order) -> the slot of each; ids whose slot changes hands restart it"""
        slot = [int(np.flatnonzero(self.ids == i)[0]) if (self.ids == i).any() else -1 for i in ids]
        taken = np.zeros(self.P, bool)
        taken[[s for s in slot if s >= 0]] = True
        for q, i in enumerate(ids):
            if slot[q] >= 0:
                continue
            free = np.flatnonzero((self.ids < 0) & ~taken)
            if free.size:
                s = int(free[0])
            else:
                cand = np.flatnonzero(~taken)
                s = int(cand[np.argmin(self.seen[cand])])          # argmin: the lowest slot on a tie
            slot[q] = s
            taken[s] = True
            self.ids[s] = i
            self.fresh[s] = True
        self.seen[taken] = tick
        return slot


def inputs(preds, maxvals, slot_active, W, H):
    """decoded COCO keypoints (n, 17, 2) and scores (n, 17) -> H36M keypoints after the repair (n, 17, 2), H36M scores
    (n, 17), the normalised input rows (n, 17, 2) and active (n,): slot_active and keep and valid; zero where inactive"""
    kp = np.asarray(preds, F32).reshape(-1, 17, 2)
    sc = np.asarray(maxvals, F32).reshape(-1, 17)
    h, where = coco_h36m(kp)
    valid = np.zeros(len(kp), bool)
    valid[where] = True
    keep = (kp != 0).reshape(len(kp), -1).any(1)
    n = np.zeros_like(sc)
    for hj, cj in _COCO_TO_H36M.items():
        n[:, hj] = sc[:, cj]
    n[:, 0] = (sc[:, 11] + sc[:, 12]) / F32(2)
    n[:, 8] = (sc[:, 5] + sc[:, 6]) / F32(2)
    n[:, 7] = (n[:, 0] + n[:, 8]) / F32(2)
    n[:, 10] = (((sc[:, 1] + sc[:, 2]) + sc[:, 3]) + sc[:, 4]) / F32(4)
    low = n[:, [2, 3, 5, 6]] < F32(0.3)
    code = low[:, 0] * 1 + low[:, 1] * 2 + low[:, 2] * 4 + low[:, 3] * 8
    rep = h.copy()
    for c, dst, src in ((15, [2, 3, 5, 6], [1, 1, 4, 4]), (11, [2, 3, 6], [1, 1, 5]), (14, [3, 5, 6], [2, 4, 4]),
                        (10, [3, 6], [2, 5]), (2, [3], [2]), (8, [6], [5])):
        m = code == c
        rep[np.ix_(m, dst)] = h[m][:, src]
    active = np.asarray(slot_active, bool) & keep & valid
    rep[~active] = 0
    n[~active] = 0
    x = (rep / F32(W) * F32(2)).astype(np.float64) - np.array([1.0, float(F32(H)) / float(F32(W))])
    x = x.astype(F32)
    x[~active] = 0
    return rep, n, x, active


def place(world, kpts, active, C, P, W):
    """revise_skes_real_time of each camera's active slots of world (C * P, 17, 3) with their keypoints (C * P, 17, 2);
    inactive slots zero"""
    world = np.asarray(world, F32).reshape(C, P, 17, 3)
    kpts = np.asarray(kpts, F32).reshape(C, P, 17, 2)
    act = np.asarray(active, bool).reshape(C, P)
    out = np.zeros_like(world)
    r = F32(500. * (W / 1920))
    for c in range(C):
        a = act[c]
        if not a.any():
            continue
        k = kpts[c, a]
        m = ((((k[:, 1] + k[:, 4]) + k[:, 11]) + k[:, 14]) / F32(4))
        o = world[c, a].copy()
        o[:, :, 0] -= ((m[:, 0] - F32(3 * W / 5)) / r)[:, None]
        o[:, :, 1] += ((m[:, 1] - F32(W / 5)) / r)[:, None]
        o[:, :, 2] -= o[:, :, 2].min()
        out[c, a] = o
    return out.reshape(C * P, 17, 3)
