"""CPU: the indices of a peek (SequenceBook.peek, the bookkeeping of PoseStream.peek) equal `end()` followed by one
`advance()` per peeked push on a deep copy of the book, for live, ending, idle, freshly reset streams and streams
shorter than the latency; the book itself is unchanged.  They also equal the peek reference's indices
(tests/peekref.py), an independent bookkeeping driven by the same events."""
import copy

import numpy as np
import pytest

from gast_b200.realtime import SequenceBook
import delayedref as D
import peekref as P


def script(book, K):
    """the scripted peek: end every live stream, then K pushes"""
    ref = copy.deepcopy(book)
    ref.end()
    return np.stack([ref.advance()[2] for _ in range(K)], 1)


def state(book):
    return book.fresh.copy(), book.length.copy(), book.left.copy()


def same(a, b):
    return all(np.array_equal(u, v) for u, v in zip(a, b))


@pytest.mark.parametrize('latency', [1, 7, 13, 121])
def test_peek_equals_end_and_advance_script(latency):
    rng = np.random.default_rng(latency)
    n = 10
    book = SequenceBook(n, latency)
    for it in range(80):
        # random events between pushes: resets and ends (also of fresh, ending and idle streams)
        for _ in range(int(rng.integers(0, 3))):
            ss = list(rng.choice(n, size=int(rng.integers(1, n + 1)), replace=False))
            getattr(book, 'reset' if rng.random() < 0.5 else 'end')(None if rng.random() < 0.1 else ss)
        for K in sorted({1, max(1, latency // 2), latency, int(rng.integers(1, latency + 1))}):
            before = state(book)
            got = book.peek(K)
            assert same(state(book), before), (it, K)
            want = script(book, K)
            assert got.shape == (n, K) and np.array_equal(got, want), (it, K)
        if rng.random() < 0.3:
            book.advance_many(int(rng.integers(1, 2 * latency + 2)))
        else:
            book.advance()


def test_every_kind_of_stream():
    """live (long and shorter than the latency), ending, idle, freshly reset and never pushed streams, by hand"""
    lat, K = 4, 4
    book = SequenceBook(6, lat)
    book.advance_many(6)                                     # every stream live with 6 frames
    book.end([1])                                            # 1: ending
    book.advance()                                           # 0, 2..5: 7 frames; 1: 3 pushes left
    book.end([2])
    book.advance_many(5)                                     # 2: idle
    book.reset([4])
    book.advance_many(2)                                     # 4: live with 2 frames (< latency)
    book.reset([3])                                          # 3: freshly reset, nothing pushed
    book.reset([5])                                        # 5: reset, then ended before its first frame
    book.end([5])
    got = book.peek(K)
    assert book.length[0] == 14 and got[0].tolist() == [10, 11, 12, 13]
    assert got[1].tolist() == [-1] * K                       # its tail was returned by the pushes
    assert got[2].tolist() == [-1] * K
    assert got[3].tolist() == [-1] * K
    assert got[4].tolist() == [-1, -1, 0, 1]
    assert got[5].tolist() == [-1] * K
    assert np.array_equal(got, script(book, K))
    book.end([0])
    book.advance()                                           # 0: ending, 3 pushes left
    assert book.peek(K)[0].tolist() == list(range(book.length[0] - 3, book.length[0])) + [-1]


def test_matches_peek_reference_bookkeeping():
    """the delayed-stream events of a case, replayed on a book, peeked at every push point"""
    events = ((3, 'end', (1,)), (5, 'reset', (1,)), (9, 'reset', (2, 3)), (9, 'end', (3,)), (16, 'end', (0, 2)),
              (17, 'reset', (0,)), (30, 'end', None), (38, 'reset', (1,)))
    case = D.Case(17, (3, 3, 3), 0, 4, 45, 0, events, 1, False, False)
    lat = D.latency(case.fw, False)
    book = SequenceBook(case.n, lat)
    for t in range(case.T + 1):
        for tt, kind, ss in case.events:
            if tt == t:
                getattr(book, kind)(None if ss is None else list(ss))
        for K in (1, 5, lat):
            want = np.stack([P.expected_index(case, s, t, K) for s in range(case.n)])
            assert np.array_equal(book.peek(K), want), (t, K)
        if t < case.T:
            book.advance()


def test_bad_k():
    book = SequenceBook(2, 3)
    with pytest.raises(ValueError):
        book.peek(0)
