"""numpy restatement of the delayed live tick's per-slot bookkeeping (csrc/live.cuh, gast_live_delayed_inputs /
_end / _place; DESIGN.md §8.11), vectorised over slots:
  Sequences.tick   one tick: which sequences end (restart, gap), their tails' frame positions, each pushed slot's
                   final and provisional frame positions and the ring position its newest frame is written to;
  Sequences.end    end(cameras): the tails of every pending sequence of the listed cameras;
  place_groups     the three placement groups: final and provisional poses placed per camera over the group's slots
                   (liveref.place), each tail row on its own.
Positions are frame positions within a slot's current (or ended) sequence, -1 where nothing is due."""
import numpy as np

import liveref as LR

F32 = np.float32


class Sequences(object):
    """n slots of a tick with latency `latency` (>= 1), provisional lookahead (None or 0 .. latency - 1) and max_gap
    (None or >= 0)"""

    def __init__(self, n, latency, lookahead=None, max_gap=None):
        self.n, self.latency, self.lookahead, self.max_gap = n, latency, lookahead, max_gap
        self.R = latency + 1
        self.id = np.full(n, -1, np.int64)       # the SORT id of the current sequence
        self.last = np.full(n, -1, np.int64)     # the tick of the last push
        self.len = np.zeros(n, np.int64)         # frames of the current sequence
        self.need = np.ones(n, bool)             # the slot book's restart flag

    def reset(self, slots):
        self.id[slots], self.last[slots], self.len[slots], self.need[slots] = -1, -1, 0, True

    def _tails(self, ending):
        """-> (n, latency) positions of the ending slots' pending frames (held push k returns frame len - latency + k)"""
        k = np.arange(self.latency)[None, :]
        pos = np.where(ending[:, None], self.len[:, None] - self.latency + k, -1)
        return np.where(pos >= 0, pos, -1)

    def tick(self, t, active, ids, restart):
        """tick t: active (n,) the slots that push (slot active, keep and valid), ids (n,) the slot book's ids and
        restart (n,) the slots gast_live_slots marked to restart this tick (a new id took them) -> dict of the tick's
        bookkeeping; updates the state"""
        active = np.asarray(active, bool)
        self.need |= np.asarray(restart, bool)
        pending = self.len >= 1
        gap = ~active & pending & (self.max_gap is not None) & (t - self.last > (self.max_gap or 0))
        ending = pending & (gap | (active & self.need))
        out = dict(ending=ending, tail=self._tails(ending), tail_ids=np.where(ending, self.id, -1),
                   fresh=active & self.need)
        start = active & self.need
        self.id[start] = np.asarray(ids, np.int64)[start]
        self.len[start] = 0
        self.len[active] += 1
        self.last[active] = t
        self.need[active] = False
        self.len[gap] = 0
        self.need[gap] = True
        newest = self.len - 1
        out['final'] = np.where(active & (newest - self.latency >= 0), newest - self.latency, -1)
        L = self.lookahead
        out['now'] = None if L is None else np.where(active & (newest - L >= 0), newest - L, -1)
        out['ring'] = np.where(active, newest % self.R, -1)
        return out

    def end(self, cameras, P):
        """end(cameras): the listed cameras' slots with frames pending -> (ending (n,), tail (n, latency) positions,
        tail_ids (n,)); then those cameras restart"""
        cams = np.zeros(self.n // P, bool)
        cams[list(cameras)] = True
        ending = np.repeat(cams, P) & (self.len >= 1)
        out = ending, self._tails(ending), np.where(ending, self.id, -1)
        self.reset(np.flatnonzero(np.repeat(cams, P)))
        return out


def ring_slot(pos, R):
    """the ring position of frame position pos (-1 where pos < 0)"""
    pos = np.asarray(pos)
    return np.where(pos >= 0, pos % R, -1)


def place_groups(world, kp, member, C, P, W):
    """one group placed as gast_live_delayed_place places the final or the provisional poses: world (C * P, 17, 3) the
    group's world poses, kp (C * P, 17, 2) the keypoints of each pose's own frame, member (C * P,) -> placed poses, zero
    outside the group (revise_skes_real_time over each camera's members)"""
    return LR.place(world, kp, member, C, P, W)


def place_tail(world, kp, due, W):
    """the tail rows: world (m, 17, 3) and kp (m, 17, 2) of each row's frame, due (m,) -> each due row placed on its
    own (revise_skes_real_time of that one pose), zero elsewhere"""
    world = np.asarray(world, F32)
    out = np.zeros_like(world)
    for i in np.flatnonzero(due):
        out[i] = LR.place(world[i:i + 1], kp[i:i + 1], [True], 1, 1, W)[0]
    return out
