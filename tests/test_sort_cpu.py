"""CPU checks of tests/sortref.py, the restatement the device tracker (csrc/track.cuh) is held to: its assignment equals
scipy's linear_sum_assignment on tie-heavy matrices, and its Sort equals the reference's outputs
(tests/golden/sort.npz) bit for bit."""
import os
import sys

import numpy as np
import pytest
from scipy.optimize import linear_sum_assignment

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sortref as R                                                 # noqa: E402
from conftest import load_golden                                    # noqa: E402


def _matrices(count, seed):
    rng = np.random.default_rng(seed)
    for k in range(count):
        nr, nc = rng.integers(0, 9, 2)
        kind = k % 5
        if kind == 0:
            m = np.zeros((nr, nc))
        elif kind == 1:
            m = rng.integers(0, 3, (nr, nc)).astype(np.float64)
        elif kind == 2:
            m = -((rng.random((nr, nc)) < 0.2) * rng.integers(1, 4, (nr, nc))) / 4.0
        elif kind == 3:
            m = -rng.random((nr, nc)).astype(np.float32)          # SORT's -iou, float32
            m[rng.random((nr, nc)) < 0.6] = 0
        else:
            m = np.full((nr, nc), -0.5)
            m[rng.random((nr, nc)) < 0.5] = -0.0
        yield m


def test_lsap_equals_scipy_on_tie_heavy_matrices():
    n = 0
    for m in _matrices(4000, 1):
        a, b = linear_sum_assignment(m)
        c, d = R.lsap(m)
        assert np.array_equal(a, c) and np.array_equal(b, d), m
        n += 1
    for shape in ((0, 4), (4, 0), (0, 0)):
        c, d = R.lsap(np.zeros(shape))
        assert c.size == 0 and d.size == 0
    assert n == 4000


def test_lsap_refuses_what_scipy_refuses():
    for bad in (np.array([[0., np.nan]]), np.array([[-np.inf, 0.]])):
        with pytest.raises(ValueError):
            linear_sum_assignment(bad)
        with pytest.raises(ValueError):
            R.lsap(bad)


def test_restated_sort_equals_the_reference():
    g = load_golden('sort')
    meta = g['meta']['scenarios']
    scen = R.scenarios()
    assert set(scen) == set(meta)
    for name, (max_age, min_hits, frames) in scen.items():
        m = meta[name]
        assert (m['max_age'], m['min_hits'], m['frames']) == (max_age, min_hits, len(frames))
        s = R.Sort(max_age, min_hits)
        counts, rows = [], []
        stop = m['raised']['frame'] if m['raised'] else len(frames)
        for t in range(stop):
            r = s.update(frames[t])
            counts.append(len(r))
            rows.append(r)
        if m['raised']:
            err = {'ZeroDivisionError': ZeroDivisionError, 'ValueError': ValueError}[m['raised']['error']]
            with pytest.raises(err):
                s.update(frames[stop])
        assert np.array_equal(np.array(counts, np.int32), g['%s_counts' % name]), name
        got = np.concatenate(rows) if rows else np.empty((0, 5))
        want = g['%s_rows' % name]
        assert got.shape == want.shape and np.array_equal(got.view(np.uint64), want.view(np.uint64)), name


def test_scenarios_cover_the_cases():
    """the goldens reach the x[6] guard, ties with more detections than trackers, id-swapping crossings and warm-up"""
    scen = R.scenarios()
    fired = []
    orig = R.Track.predict

    def predict(self):
        fired.append(bool(self.kf.x[6] + self.kf.x[2] <= 0))
        return orig(self)

    R.Track.predict = predict
    try:
        R.run(scen['shrink'][2], *scen['shrink'][:2])
    finally:
        R.Track.predict = orig
    assert any(fired)
    frames = scen['many_ties'][2]
    assert sum(len(f) > 3 for f in frames) > 10
    out = R.run(scen['warmup'][2], *scen['warmup'][:2])
    assert [len(o) for o in out][:3] == [1, 2, 3]
    assert scen['five_col'][2][0].shape[1] == 5


def test_packing_of_frames():
    frames = [R._boxes([[0, 0, 100, 100]]), np.zeros((0, 4), np.float32), R._boxes([[1, 2, 3, 4], [5, 6, 7, 8]])]
    b, n = R.pack(frames)
    assert b.shape == (3, 2, 4) and list(n) == [1, 0, 2] and not b[1].any() and not b[0, 1].any()
