"""CPU: the fp64 delayed-stream reference of tests/delayedref.py reproduces what the unmodified reference computes for
whole sequences (the delayed_* goldens: UnchunkedGenerator + tools.inference.evaluate, with and without test-time
augmentation); and the host-side bookkeeping of gast_b200.realtime.PoseStream (SequenceBook: fresh and hold masks,
returned indices) equals recomputing every pose from its own generator window, with a stub in place of the network
(the network itself has no CPU path)."""
import numpy as np
import pytest
import torch

from conftest import golden_names, load_golden
from gast_b200.realtime import SequenceBook
import delayedref as D

# max |y_golden - y64| / max |y64| measured over the five goldens: 6.8e-7 to 3.0e-6 (the reference's fp32 rounding;
# the largest is the 128-channel causal model), relative L2 4.7e-7 to 2.3e-6
GOLDEN_BAR = 1e-5


def test_delayed_goldens_present():
    assert golden_names('delayed_') == ['delayed_17_3333_c64_aug', 'delayed_17_333_c128_causal_aug',
                                        'delayed_17_333_c32', 'delayed_17_333_c32_aug', 'delayed_19_333_c32_aug']


@pytest.mark.parametrize('name', golden_names('delayed_'))
def test_reference_matches_delayed_goldens(name):
    g = load_golden(name)
    meta = g['meta']
    case = D.Case(meta['J'], tuple(meta['filter_widths']), meta['channels'], 1, 1, 0, (), meta['seed'],
                  meta['causal'], meta['augment'])
    m = D.module(case)
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == meta['keys']
    assert (meta['pad'], meta['causal_shift']) == D.pad_shift(case.fw, case.causal)
    lists = (meta['kps_left'], meta['kps_right'], meta['joints_left'], meta['joints_right'])
    assert lists == D.symmetry(case.J)
    cuts = np.cumsum([0] + meta['lengths'])
    seqs = [g['x'][a:b] for a, b in zip(cuts[:-1], cuts[1:])]
    y64 = np.concatenate(D.sequence_poses(seqs, case.J, case.fw, case.causal, case.augment, lists, m.state_dict()))
    mx = float(np.abs(g['y'] - y64).max() / np.abs(y64).max())
    l2 = float(np.linalg.norm(g['y'] - y64) / np.linalg.norm(y64))
    assert mx <= GOLDEN_BAR and l2 <= GOLDEN_BAR, (mx, l2)


class WindowProbe(object):
    """Stands in for the network: 'lifts' a window of rf frames to a weighted sum over its frames, so that any
    mistake in the order, the padding or the delay of the window changes the result."""

    def __init__(self, rf):
        self.w = np.arange(1, rf + 1, dtype=np.float64) ** 1.5

    def __call__(self, win):                                   # (..., rf, J, 2) -> (..., J, 2)
        return np.tensordot(win, self.w, axes=([-3], [0])).transpose(tuple(range(win.ndim - 3)) + (-2, -1))


def drive(case):
    """push the frames of `case` through SequenceBook and a model of the library's input history (fill-fresh, hold
    = re-append the newest frame) of rf frames; the probe of each push's window is its output.
    -> (outputs (n, T, J, 2), index (n, T))"""
    rf = D.S.receptive_field(case.fw)
    lat = D.latency(case.fw, case.causal)
    book = SequenceBook(case.n, lat)
    probe = WindowProbe(rf)
    x = D.frames(case).astype(np.float64)
    hist = np.zeros((case.n, rf, case.J, 2))
    outs, idx = [], []
    for t in range(case.T):
        for tt, kind, ss in case.events:
            if tt == t:
                getattr(book, kind)(None if ss is None else list(ss))
        fresh, hold, index = book.advance()
        assert not (fresh & hold).any()
        row = x[t].copy()
        row[hold] = np.nan                                     # the rows of held streams are ignored
        for s in range(case.n):
            if fresh[s]:
                hist[s] = row[s]
            else:
                new = hist[s, -1].copy() if hold[s] else row[s]
                hist[s] = np.concatenate([hist[s, 1:], new[None]])
        outs.append(probe(hist))
        idx.append(index)
    return np.stack(outs, 1), np.stack(idx, 1)


BOOK_CASES = [
    # non-causal 27 frames (latency 13): ends on a stream shorter than the latency, reset during a pending tail, end
    # and reset on consecutive pushes, end of every stream, idle streams, a reset of a pending-fresh stream
    D.Case(17, (3, 3, 3), 0, 4, 90, 0, ((5, 'end', (1,)), (9, 'reset', (1,)), (20, 'end', (0,)), (21, 'reset', (0,)),
                                        (30, 'end', (2,)), (38, 'reset', (2,)), (40, 'end', None),
                                        (46, 'end', (3,)), (60, 'reset', (1, 3)), (60, 'end', (3,)),
                                        (70, 'reset', None), (71, 'reset', (2,)), (80, 'end', (0, 1))), 1, False,
           False),
    # causal: latency 0, end makes a stream idle at once
    D.Case(17, (3, 3), 0, 3, 30, 0, ((4, 'end', (1,)), (10, 'reset', (1,)), (12, 'end', None), (20, 'reset', (0, 2))),
           2, True, False),
    # a first width of 5 and a 5-tap stage (latency 37), a sequence of one frame
    D.Case(16, (5, 5, 3), 0, 3, 130, 0, ((1, 'end', (2,)), (3, 'reset', (2,)), (50, 'end', (0,)), (100, 'end', (1,))),
           3, False, False),
]


@pytest.mark.parametrize('k', range(len(BOOK_CASES)))
def test_bookkeeping_equals_per_frame_windows(k):
    case = BOOK_CASES[k]
    rf = D.S.receptive_field(case.fw)
    pad, shift = D.pad_shift(case.fw, case.causal)
    probe = WindowProbe(rf)
    x = D.frames(case).astype(np.float64)
    got, idx = drive(case)
    assert np.isfinite(got[idx >= 0]).all()
    returned = 0
    for s in range(case.n):
        assert np.array_equal(idx[s], D.expected_index(case, s)), s          # two independent bookkeepings
        for t0, te, cut in D.sequences(case, s):
            padded = D.generator_batch(x[t0:te, s], pad, shift, False, [], [])[0]
            for j in range(te - t0):
                p = t0 + j + pad - shift
                if p >= cut:
                    continue
                want = probe(padded[j:j + rf])
                assert np.abs(got[s, p] - want).max() <= 1e-9 * np.abs(want).max(), (s, t0, j)
                returned += 1
    assert returned == int((idx >= 0).sum())                                  # nothing returned that is not due
