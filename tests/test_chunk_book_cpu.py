"""CPU: SequenceBook.advance_many (the bookkeeping of PoseStream.push_frames) equals K calls of advance(), with end()
inserted before push valid[s] of every live stream whose valid[s] < K, over random reset / end scripts."""
import copy

import numpy as np
import pytest

from gast_b200.realtime import SequenceBook


def script(book, K, valid):
    """the K-step advance() / end() script advance_many must reproduce"""
    fr, ho, ix = [], [], []
    ends = {}
    if valid is not None:
        live = book.left < 0
        for s in np.flatnonzero(live & (np.asarray(valid) < K)):
            ends.setdefault(int(valid[s]), []).append(int(s))
    for k in range(K):
        if k in ends:
            book.end(ends[k])
        f, h, i = book.advance()
        fr.append(f)
        ho.append(h)
        ix.append(i)
    return fr[0], np.stack(ho, 1), np.stack(ix, 1)


def same_state(a, b):
    return (np.array_equal(a.fresh, b.fresh) and np.array_equal(a.length, b.length)
            and np.array_equal(a.left, b.left))


@pytest.mark.parametrize('latency', [0, 1, 7, 121])
def test_advance_many_equals_advance_script(latency):
    rng = np.random.default_rng(latency)
    n = 12
    book = SequenceBook(n, latency)
    Ks = [1, 2, 3, 7, 64, 300, 1, 5, 121, 122, 250]
    for it in range(60):
        # random events between calls: resets and ends of random streams (also on fresh, ending and idle streams)
        for _ in range(int(rng.integers(0, 3))):
            ss = list(rng.choice(n, size=int(rng.integers(1, n + 1)), replace=False))
            getattr(book, 'reset' if rng.random() < 0.5 else 'end')(None if rng.random() < 0.1 else ss)
        K = Ks[it % len(Ks)] if it % 3 else int(rng.integers(1, 301))
        mode = it % 4
        if mode == 0:
            valid = None
        else:
            # 0, mid-chunk and K, mixed over the streams
            valid = rng.choice([0, int(rng.integers(0, K + 1)), K], size=n)
        ref = copy.deepcopy(book)
        want = script(ref, K, valid)
        got = book.advance_many(K, valid)
        for g, w, what in zip(got, want, ('fresh', 'hold', 'index')):
            assert g.shape == w.shape and np.array_equal(g, w), (it, K, what, valid)
        assert same_state(book, ref), it


def test_every_valid_on_one_stream():
    """every end position 0..K on a fresh, a live, an ending and an idle stream"""
    K, lat = 9, 4
    for v in range(K + 1):
        book = SequenceBook(4, lat)
        book.advance_many(6)                                  # all live, 6 frames
        book.reset([0])                                       # fresh
        book.end([2])                                         # ending
        book.end([3])
        book.advance_many(5)                                  # 3 idle after its tail
        book.reset([0])
        ref = copy.deepcopy(book)
        want = script(ref, K, np.full(4, v))
        got = book.advance_many(K, np.full(4, v))
        for g, w in zip(got, want):
            assert np.array_equal(g, w), v
        assert same_state(book, ref), v


def test_bad_arguments():
    book = SequenceBook(3, 2)
    with pytest.raises(ValueError):
        book.advance_many(0)
    with pytest.raises(ValueError):
        book.advance_many(4, [0, 5, 1])
    with pytest.raises(ValueError):
        book.advance_many(4, [0, 1])
    with pytest.raises(ValueError):
        book.advance_many(4, [0, -1, 1])
