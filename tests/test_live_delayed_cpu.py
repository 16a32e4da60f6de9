"""The numpy restatement of the delayed live tick's bookkeeping (tests/livedelayedref.py) against realtime.SequenceBook
on hand-built id and activity sequences: which frame each final, provisional and tail row belongs to (the book's
`advance` / `peek` indices of the composition peek(latency, ending) -> reset(ending) -> push(active) ->
peek(latency - L, active)), when a tail is due (restart, gap, end), the ring positions, and the placement groups
against tests/preprocessref.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import livedelayedref as LD                                         # noqa: E402
import liveref as LR                                                # noqa: E402
import preprocessref as PR                                          # noqa: E402
from gast_b200.realtime import SequenceBook                         # noqa: E402

F32 = np.float32


def _schedule(n, T, seed, p_active=0.7, p_new=0.05):
    """T ticks of n slots: activity, the slot book's ids and its restart marks (a new id takes the slot)"""
    rng = np.random.default_rng(seed)
    ids = np.full(n, -1, np.int64)
    nxt = 1
    out = []
    for _ in range(T):
        act = rng.random(n) < p_active
        restart = np.zeros(n, bool)
        for s in range(n):
            if (ids[s] < 0 and act[s]) or rng.random() < p_new:
                ids[s], nxt, restart[s] = nxt, nxt + 1, True
        out.append((act, ids.copy(), restart))
    return out


def _composition(book, latency, L, act, ending, fresh):
    """the composition's indices: peek(latency, ending) -> reset(ending and the restarting slots) -> push(active) ->
    peek(latency - L, active)"""
    n = book.n
    tail = np.full((n, latency), -1, np.int64)
    if ending.any():
        tail[ending] = book.peek(latency, streams=np.flatnonzero(ending))
    if (ending | fresh).any():
        book.reset(np.flatnonzero(ending | fresh))
    final = np.full(n, -1, np.int64)
    now = np.full(n, -1, np.int64)
    s = np.flatnonzero(act)
    if s.size:
        final[s] = book.advance(streams=s)[2]
        if L is not None:
            now[s] = book.peek(latency - L, streams=s)[:, -1]
    return tail, final, now


@pytest.mark.parametrize('latency,L,max_gap', [(1, None, None), (1, 0, 0), (13, None, None), (13, 0, 2),
                                               (13, 12, None), (40, 5, 3), (4, 3, 0)])
def test_positions_equal_the_sequence_book(latency, L, max_gap):
    n, T = 6, 300
    ref = LD.Sequences(n, latency, L, max_gap)
    book = SequenceBook(n, latency)
    tails = 0
    for t, (act, ids, restart) in enumerate(_schedule(n, T, seed=latency * 7 + (max_gap or 0))):
        pre_len = ref.len.copy()
        out = ref.tick(t, act, ids, restart)
        ending = out['ending']
        tail, final, now = _composition(book, latency, L, act, ending, out['fresh'])
        np.testing.assert_array_equal(out['tail'], tail)
        assert (out['tail_ids'][ending] >= 1).all() and (out['tail_ids'][~ending] == -1).all()
        assert (pre_len[ending] >= 1).all()
        tails += int(ending.sum())
        np.testing.assert_array_equal(out['final'], final)
        if L is not None:
            np.testing.assert_array_equal(out['now'], now)
        np.testing.assert_array_equal(out['ring'], np.where(act, (ref.len - 1) % (latency + 1), -1))
    assert tails > 5


def test_tails_are_due_on_restart_gap_and_end():
    lat = 3
    ref = LD.Sequences(2, lat, None, max_gap=1)
    ids = np.array([1, 2])
    for t in range(4):
        out = ref.tick(t, [True, True], ids, [t == 0, t == 0])
        assert not out['ending'].any()
    out = ref.tick(4, [True, False], ids, [False, False])          # slot 1 misses one tick: within the gap
    assert not out['ending'].any()
    out = ref.tick(5, [True, False], ids, [False, False])          # two ticks missed: more than max_gap = 1
    assert out['ending'].tolist() == [False, True] and out['tail'][1].tolist() == [1, 2, 3]
    assert out['tail_ids'].tolist() == [-1, 2]
    out = ref.tick(6, [True, True], np.array([3, 2]), [True, False])   # a new id restarts slot 0; slot 1 starts anew
    assert out['ending'].tolist() == [True, False] and out['tail'][0].tolist() == [3, 4, 5]
    assert out['fresh'].tolist() == [True, True] and out['tail_ids'].tolist() == [1, -1]
    assert out['final'].tolist() == [-1, -1]
    ending, tail, tail_ids = ref.end([0], 1)
    assert ending.tolist() == [True, False] and tail[0].tolist() == [-1, -1, 0] and tail_ids.tolist() == [3, -1]
    assert ref.len.tolist() == [0, 1]
    ending, tail, _ = ref.end([0], 1)
    assert not ending.any()


def test_no_gap_rule_joins_the_frames_across_gaps():
    ref = LD.Sequences(1, 2, None, None)
    pos = []
    for t in range(40):
        out = ref.tick(t, [t % 5 != 3], [7], [t == 0])
        assert not out['ending'].any()
        pos.append(int(out['final'][0]))
    got = [p for p in pos if p >= 0]
    assert got == list(range(len(got))) and len(got) == 32 - 2


def test_ring_positions_keep_the_pending_frames():
    """the ring of latency + 1 frames holds every frame a final, provisional or tail row reads until the placement
    has read it, written after the reads"""
    lat, R = 4, 5
    ref = LD.Sequences(1, lat, 0, None)
    ring = np.full(R, -1)
    for t, (act, restart) in enumerate([(True, True)] * 9 + [(False, False)] * 2 + [(True, True)] + [(True, False)] * 3):
        out = ref.tick(t, [act], [t // 11 + 1], [restart])
        for pos in list(out['tail'][0]) + [out['final'][0]]:
            if pos >= 0:
                assert ring[pos % R] == pos
        if act:
            ring[out['ring'][0]] = ref.len[0] - 1
    assert LD.ring_slot([-1, 0, 4, 5, 13], R).tolist() == [-1, 0, 4, 0, 3]


def test_placement_groups_equal_revise_skes_real_time():
    rng = np.random.default_rng(5)
    C, P, W, lat = 3, 2, 640, 3
    world = rng.standard_normal((C * P, 17, 3)).astype(F32)
    kp = rng.uniform(0, W, (C * P, 17, 2)).astype(F32)
    member = np.array([True, False, True, True, False, False])
    got = LD.place_groups(world, kp, member, C, P, W)
    for c in range(C):
        m = member[c * P:(c + 1) * P]
        if m.any():
            want = PR.revise_skes_real_time(world[c * P:(c + 1) * P][m], kp[c * P:(c + 1) * P][m], W)
            np.testing.assert_array_equal(got[c * P:(c + 1) * P][m], want)
    assert (got[~member] == 0).all()
    tw = rng.standard_normal((C * P * lat, 17, 3)).astype(F32)
    tk = rng.uniform(0, W, (C * P * lat, 17, 2)).astype(F32)
    due = rng.random(C * P * lat) < 0.5
    tail = LD.place_tail(tw, tk, due, W)
    for i in range(C * P * lat):
        if due[i]:
            np.testing.assert_array_equal(tail[i], PR.revise_skes_real_time(tw[i:i + 1], tk[i:i + 1], W)[0])
        else:
            assert (tail[i] == 0).all()
    # with latency 0 the final group is gast_live_place's rule: the active slots of each camera together
    np.testing.assert_array_equal(LD.place_groups(world, kp, member, C, P, W), LR.place(world, kp, member, C, P, W))
