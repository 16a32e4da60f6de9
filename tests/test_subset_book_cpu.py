"""CPU: SequenceBook with `streams` (the bookkeeping of PoseStream's subset calls) equals independent one-stream books
stepped only on the calls their stream takes part in, over random schedules of advances, chunks, peeks, resets and
ends; and the host validation of `streams`."""
import copy

import numpy as np
import pytest

from gast_b200.realtime import SequenceBook


def same(a, b):
    return (np.array_equal(a.fresh, b.fresh) and np.array_equal(a.length, b.length)
            and np.array_equal(a.left, b.left))


@pytest.mark.parametrize('latency', [0, 1, 7, 40])
def test_subset_calls_equal_one_stream_books(latency):
    rng = np.random.default_rng(100 + latency)
    n = 9
    book = SequenceBook(n, latency)
    solo = [SequenceBook(1, latency) for _ in range(n)]
    for it in range(300):
        if rng.random() < 0.3:                               # events between calls, on random streams
            ss = [int(s) for s in rng.choice(n, size=int(rng.integers(1, 4)), replace=False)]
            kind = 'reset' if rng.random() < 0.5 else 'end'
            getattr(book, kind)(ss)
            for s in ss:
                getattr(solo[s], kind)()
        m = int(rng.choice([1, 2, n // 2, n]))
        sel = rng.permutation(n)[:m]
        op = it % 4
        if op == 0:
            got = book.advance(streams=sel)
            want = [solo[s].advance() for s in sel]
            for g, k in zip(got, range(3)):
                assert np.array_equal(g, np.concatenate([w[k] for w in want])), (it, k)
        elif op in (1, 2):
            K = int(rng.choice([1, 2, 5, 13, 41]))
            valid = None if op == 1 else rng.integers(0, K + 1, size=m)
            got = book.advance_many(K, valid, streams=sel)
            want = [solo[s].advance_many(K, None if valid is None else valid[i:i + 1]) for i, s in enumerate(sel)]
            for k in range(3):
                assert np.array_equal(got[k], np.concatenate([w[k] for w in want])), (it, k)
        else:
            K = int(rng.integers(1, latency + 1)) if latency else 1
            before = copy.deepcopy(book)
            got = book.peek(K, streams=sel)
            assert same(book, before), it                    # a peek changes nothing
            assert np.array_equal(got, np.concatenate([solo[s].peek(K) for s in sel])), it
        for s in range(n):
            assert (book.fresh[s], book.length[s], book.left[s]) == \
                (solo[s].fresh[0], solo[s].length[0], solo[s].left[0]), (it, s)


def test_unlisted_streams_unchanged():
    book = SequenceBook(5, 3)
    book.advance_many(4)
    book.end([1])
    before = copy.deepcopy(book)
    book.advance_many(6, streams=[3, 0])
    book.advance(streams=[4])
    for s in (1, 2):
        assert (book.fresh[s], book.length[s], book.left[s]) == (before.fresh[s], before.length[s], before.left[s])


def test_all_streams_in_order_equals_no_streams():
    a, b = SequenceBook(4, 2), SequenceBook(4, 2)
    for K, valid in ((3, None), (1, None), (5, [5, 0, 2, 5]), (2, None)):
        ga = a.advance_many(K, valid)
        gb = b.advance_many(K, valid, streams=[0, 1, 2, 3])
        assert all(np.array_equal(x, y) for x, y in zip(ga, gb))
        assert same(a, b)


@pytest.mark.parametrize('bad', [[], [3], [-1], [0, 0], [1, 2, 1], [0.5], np.arange(4)])
def test_bad_streams(bad):
    book = SequenceBook(3, 2)
    before = copy.deepcopy(book)
    for call in (lambda: book.advance(streams=bad), lambda: book.advance_many(2, streams=bad),
                 lambda: book.peek(1, streams=bad)):
        with pytest.raises(ValueError, match='streams'):
            call()
    assert same(book, before)


def test_valid_has_one_value_per_listed_stream():
    book = SequenceBook(4, 2)
    with pytest.raises(ValueError):
        book.advance_many(3, [1, 2, 3, 0], streams=[0, 1])
