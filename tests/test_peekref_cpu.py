"""CPU: the fp64 peek reference of tests/peekref.py reproduces what the unmodified reference computes for the prefixes of
a sequence (the peek_* goldens: UnchunkedGenerator + tools.inference.evaluate on every prefix, with and without
test-time augmentation), and agrees with the delayed-stream reference of tests/delayedref.py wherever a peek is
final: once a sequence has ended, its peek is the tail the next pushes return."""
import numpy as np
import pytest

from conftest import golden_names, load_golden
import delayedref as D
import peekref as P

# max |y_golden - y64| / max |y64| measured over the four goldens: 6.4e-7 to 1.2e-6 (the reference's fp32 rounding),
# relative L2 3.4e-7 to 5.9e-7; the level of tests/test_delayedref_cpu.py
GOLDEN_BAR = 1e-5


def test_peek_goldens_present():
    assert golden_names('peek_') == ['peek_17_3333_c64_aug', 'peek_17_333_c32', 'peek_17_333_c32_aug',
                                     'peek_19_333_c32_aug']


def golden_case(g):
    meta = g['meta']
    return D.Case(meta['J'], tuple(meta['filter_widths']), meta['channels'], 1, len(g['x']), 0, (), meta['seed'], False,
                  meta['augment'])


@pytest.mark.parametrize('name', golden_names('peek_'))
def test_reference_matches_peek_goldens(name):
    g = load_golden(name)
    meta = g['meta']
    case = golden_case(g)
    m = D.module(case)
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == meta['keys']
    lat = D.latency(case.fw, False)
    assert meta['latency'] == lat and g['y'].shape == (len(g['prefixes']), lat, case.J, 3)
    assert (meta['kps_left'], meta['kps_right'], meta['joints_left'], meta['joints_right']) == D.symmetry(case.J)
    y64, index = P.peeks(case, g['x'][:, None], (0,), [int(p) for p in g['prefixes']], lat, m.state_dict())
    y64, index = y64[0], index[0]
    assert np.array_equal(index >= 0, np.isfinite(g['y'][..., 0, 0]))      # the rows the golden has poses for
    for q, p in enumerate(g['prefixes']):
        assert np.array_equal(index[q][index[q] >= 0], np.arange(max(0, p - lat), p))
    sel = index >= 0
    mx = float(np.abs(g['y'][sel] - y64[sel]).max() / np.abs(y64[sel]).max())
    l2 = float(np.linalg.norm(g['y'][sel] - y64[sel]) / np.linalg.norm(y64[sel]))
    assert mx <= GOLDEN_BAR and l2 <= GOLDEN_BAR, (mx, l2)


@pytest.mark.parametrize('augment', [False, True])
def test_final_peeks_equal_delayed_tails(augment):
    """after an end, a peek returns the poses the next pushes return, as the delayed reference computes them"""
    events = ((4, 'end', (2,)), (10, 'end', (0,)), (12, 'reset', (1,)), (14, 'end', (1, 3)), (25, 'end', None),
              (30, 'reset', (0,)))
    case = D.Case(17, (3, 3, 3), 16, 4, 45, 0, events, 5, False, augment)
    lat = D.latency(case.fw, False)
    x = D.frames(case)
    points = list(range(case.T + 1))
    y, index = P.peeks(case, x, tuple(range(case.n)), points, lat)
    yd, idd = D.reference(case)
    compared = 0
    for s in range(case.n):
        for q, t in enumerate(points):
            cur = P.current(case, s, t)
            if cur is None or cur[1] > t:                  # live (or nothing pushed): the peek is provisional
                continue
            for k in np.flatnonzero(index[s, q] >= 0):
                if t + k < case.T and idd[s, t + k] == index[s, q, k]:
                    assert np.abs(y[s, q, k] - yd[s, t + k]).max() <= 1e-12 * np.abs(yd[s, t + k]).max()
                    compared += 1
    assert compared > 100, compared


def test_live_peek_differs_from_final():
    """a live stream's peek is provisional: it is not the pose the stream returns once the sequence goes on"""
    case = D.Case(17, (3, 3, 3), 16, 1, 40, 0, (), 6, False, False)
    lat = D.latency(case.fw, False)
    x = D.frames(case)
    y, index = P.peeks(case, x, (0,), [20], lat)
    yd, idd = D.reference(case)
    assert index[0, 0].tolist() == list(range(20 - lat, 20))
    # the first row sees the right padding only at its window's last frame; the last row is half padding
    first = np.abs(y[0, 0, 0] - yd[0, 20]).max() / np.abs(yd[0, 20]).max()
    last = np.abs(y[0, 0, -1] - yd[0, 20 + lat - 1]).max() / np.abs(yd[0, 20 + lat - 1]).max()
    assert first > 1e-9 and last > first, (first, last)
