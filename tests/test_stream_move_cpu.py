"""CPU checks of moving streams between pools (PoseStream.export_streams / import_streams, C ABI gast_stream_export /
gast_stream_import): the numpy model of the state layout and of the move (tests/moveref.py), and the move of the
host sequence bookkeeping (SequenceBook.rows / put_rows) with live, ending, idle and fresh streams."""
import numpy as np
import pytest

from gast_b200.realtime import SequenceBook
import moveref as M


def test_snapshot_floats_of_the_flagship_geometries():
    assert M.snapshot_floats(17, 2, (3, 3, 3), 128) == 274278           # 27-frame model, 128 channels
    assert M.snapshot_floats(17, 2, (3, 3, 3, 3), 64) == 842214         # 81-frame model, 64 channels
    assert M.parts(17, 2, (3, 3, 3), 128)[0] == (1, 102)                 # 3 taps x 17 joints x 2: not a multiple of 4


def time_state(J, F, fw, ch, n, counts):
    """a state whose every ring float of stream s holds 1000 s + the time whose input the slot keeps at count
    counts[s] (the latest t < count with t = slot mod R), and whose input history holds -(1000 s + k)"""
    lay, nf = M.layout(J, F, fw, ch, n)
    st = np.full(nf, np.nan)
    for s, c in enumerate(counts):
        off, _, row = lay[0]
        st[off + s * row:off + (s + 1) * row] = -(1000 * s + np.arange(row))
        for off, R, row in lay[1:]:
            for p in range(R):
                t = c - 1 - (c - 1 - p) % R
                st[off + (p * n + s) * row:off + (p * n + s + 1) * row] = 1000 * s + t
    return st


@pytest.mark.parametrize('fw', [(3, 3, 3), (5, 3), (3, 5, 3)])
def test_snapshot_is_time_ordered_at_any_phase(fw):
    J, F, ch, n = 3, 2, 4, 4
    counts = [1, 7, 45, 100]
    st = time_state(J, F, fw, ch, n, counts)
    snap = M.export(st, J, F, fw, ch, n, [2, 0, 3], [counts[2], counts[0], counts[3]])
    for i, s in enumerate([2, 0, 3]):
        c, o = counts[s], 0
        for q, (R, row) in enumerate(M.parts(J, F, fw, ch)):
            part = snap[i, o:o + R * row].reshape(R, row)
            if q == 0:
                assert np.array_equal(part[0], -(1000 * s + np.arange(row)))
            else:
                assert np.array_equal(part[:, 0], 1000 * s + c - R + np.arange(R)), (s, q)   # oldest first
                assert (part == part[:, :1]).all()
            o += R * row
        assert o == snap.shape[1]


@pytest.mark.parametrize('fw', [(3, 3, 3), (5, 3), (3, 3, 3, 3)])
def test_import_at_another_phase_and_n_is_the_right_permutation(fw):
    """export two streams of a 5-stream state, import them into a 7-stream state at other indices and counts: the
    target slot of time t is (t - c + c') mod R, the rows of every other stream and the padding are untouched, and an
    import at the source count into a state of the same n gives back the source rows"""
    J, F, ch = 3, 2, 4
    rng = np.random.default_rng(0)
    la, na = M.layout(J, F, fw, ch, 5)
    lb, nb = M.layout(J, F, fw, ch, 7)
    a = rng.standard_normal(na)
    b = rng.standard_normal(nb)
    src, dst, ca, cb = [3, 1], [6, 0], [20, 2 ** 40 + 7], [9, 9]
    snap = M.export(a, J, F, fw, ch, 5, src, ca)
    out = M.import_(b, J, F, fw, ch, 7, dst, cb, snap)
    touched = np.zeros(nb, dtype=bool)
    for s, d, c, c2 in zip(src, dst, ca, cb):
        for q, ((oa, R, row), (ob, _, _)) in enumerate(zip(la, lb)):
            if q == 0:
                assert np.array_equal(out[ob + d * row:ob + (d + 1) * row], a[oa + s * row:oa + (s + 1) * row])
                touched[ob + d * row:ob + (d + 1) * row] = True
                continue
            for t in range(c - R, c):
                pa, pb = t % R, (t - c + c2) % R
                assert np.array_equal(out[ob + (pb * 7 + d) * row:ob + (pb * 7 + d + 1) * row],
                                      a[oa + (pa * 5 + s) * row:oa + (pa * 5 + s + 1) * row]), (q, t)
                touched[ob + (pb * 7 + d) * row:ob + (pb * 7 + d + 1) * row] = True
    assert touched.sum() == 2 * M.snapshot_floats(J, F, fw, ch)
    assert np.array_equal(out[~touched], b[~touched])
    back = M.import_(rng.standard_normal(na), J, F, fw, ch, 5, src, ca, snap)
    for s, c in zip(src, ca):
        idx = M.state_index(J, F, fw, ch, 5, s, c)
        assert np.array_equal(back[idx], a[idx])
    # the count only matters mod R_max: the same slots
    assert np.array_equal(M.state_index(J, F, fw, ch, 7, 2, 9), M.state_index(J, F, fw, ch, 7, 2, 9 + 5 * np.prod(fw)))


def driven_book(n, lat):
    """a book with a live stream, ending streams (2 and 1 pushes left), an idle one, a fresh one and one ended before
    its first frame"""
    b = SequenceBook(n, lat)
    b.advance_many(6)
    b.end([1])
    b.advance()
    b.end([2])
    b.advance()
    b.end([3])
    b.advance_many(lat + 1)                          # 3 idle; 1 and 2 too
    b.reset([1, 2, 4, 5])
    b.advance_many(4)
    b.end([1])
    b.advance()                                      # 1 ending: lat - 1 left
    b.end([2])                                       # 2 ending: lat left
    b.reset([4])                                     # 4 fresh
    b.reset([5])
    b.end([5])                                       # 5 ended before its first frame: idle
    return b


def test_book_rows_move_with_their_sequences():
    lat = 4
    a = driven_book(6, lat)
    assert a.left.tolist() == [-1, lat - 1, lat, 0, -1, 0] and a.fresh.tolist() == [False] * 4 + [True, False]
    src = [2, 0, 4, 1, 5, 3]
    dst = [5, 2, 0, 6, 3, 1]
    b = SequenceBook(8, lat)
    b.advance_many(3)
    before = b.rows([4, 7])
    b.put_rows(dst, a.rows(src))
    assert all(np.array_equal(x, y) for x, y in zip(b.rows([4, 7]), before))
    assert np.array_equal(b.peek(lat, streams=dst), a.peek(lat, streams=src))
    for K, valid in ((1, None), (3, [3, 1, 0, 3, 2, 3]), (lat + 2, None)):
        got = b.advance_many(K, valid, streams=dst)
        want = a.advance_many(K, valid, streams=src)
        for x, y in zip(got, want):
            assert np.array_equal(x, y), K
    got, want = b.advance(streams=dst), a.advance(streams=src)
    assert all(np.array_equal(x, y) for x, y in zip(got, want))
    assert all(np.array_equal(x, y) for x, y in zip(b.rows(dst), a.rows(src)))


def test_book_rows_are_copies_and_check_streams():
    a = driven_book(6, 3)
    rows = a.rows([1, 2])
    rows[2][:] = 99
    assert a.left[1] != 99
    with pytest.raises(ValueError):
        a.rows([1, 1])
    with pytest.raises(ValueError):
        a.put_rows([6], a.rows([0]))
