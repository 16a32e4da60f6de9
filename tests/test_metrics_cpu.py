"""CPU: the scoring rows of gast_pose_metrics restated in numpy (tests/metricsref.py) against the unmodified
reference's euclidean_losses, pck and auc (tests/golden/make_golden_metrics.py).  The pinned float32 order
(dx*dx + dy*dy) + dz*dz reproduces the reference's squared distances bit for bit.  The square root is IEEE-rounded
here (numpy, and __fsqrt_rn on the device); torch's CPU float32 sqrt, which the reference's numbers come from, is not
correctly rounded and lands one ulp off on a few points in a thousand.  Counts, and with them pck and auc, are the
reference's exactly, distances that land on a threshold included."""
import numpy as np
import pytest
import torch

import metricsref as MR
from conftest import load_golden

CASES = ('random', 'on_threshold', 'degenerate')
AUC = torch.linspace(0, 150, 31).tolist()


@pytest.fixture(scope='module')
def G():
    return load_golden('metrics_17')


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize('case', CASES)
def test_pinned_distance_order_is_the_references(G, case):
    p, t = G[case + '_pred'], G[case + '_tgt']
    sq = (p - t) * (p - t)
    assert np.array_equal((sq[..., 0] + sq[..., 1]) + sq[..., 2], G[case + '_dist_sq'])         # bit for bit
    d = MR.distances(p, t)
    assert d.dtype == np.float32
    assert np.array_equal(d, np.sqrt(G[case + '_dist_sq']))                                    # IEEE-rounded sqrt
    assert np.array_equal(d, np.float32(np.sqrt(G[case + '_dist_sq'].astype(np.float64))))
    off = _ulps(d, G[case + '_dist'])
    assert off.max() <= 1 and off.sum() <= 0.01 * off.size, off.sum()                          # torch's sqrt


def test_on_threshold_case_lands_on_thresholds(G):
    """the golden does test the boundary: many distances equal a threshold, where `<` decides"""
    d = G['on_threshold_dist']
    assert np.isin(d, G['thresholds']).sum() >= 100
    assert np.isin(d, np.float32(AUC)).mean() == 1.0


def test_other_grouping_differs(G):
    """dx*dx + (dy*dy + dz*dz) is not the same float32 number on ordinary data: the order has to be pinned"""
    p, t = G['random_pred'], G['random_tgt']
    sq = (p - t) * (p - t)
    other = np.sqrt(sq[..., 0] + (sq[..., 1] + sq[..., 2]))
    assert (other != G['random_dist']).sum() > 0


@pytest.mark.parametrize('case', CASES)
def test_rows_give_the_references_pck_and_auc(G, case):
    p, t = G[case + '_pred'], G[case + '_tgt']
    N, J = p.shape[:2]
    thr = list(G['thresholds']) + AUC
    rows = MR.segment_rows(p, t, [0, N], thr, procrustes=False)
    cnt = rows[0, 3 + J:]
    nthr = len(G['thresholds'])
    assert [c / (N * J) for c in cnt[:nthr]] == list(G[case + '_pck'])         # exactly, as Python floats
    auc = torch.tensor([c / (N * J) for c in cnt[nthr:]], dtype=torch.float64).mean().item()
    assert auc == float(G[case + '_auc'])
    d = G[case + '_dist'].astype(np.float64)
    assert rows[0, 0] == N
    assert np.allclose(rows[0, 1], d.mean(1).sum(), rtol=1e-7, atol=0)                          # one-ulp distances
    assert np.allclose(rows[0, 3:3 + J], d.sum(0), rtol=1e-7, atol=0)


def test_segments_partition_the_whole(G):
    """segment rows add up to the one-segment row (counts exactly), and an empty segment is a row of zeros"""
    p, t = G['random_pred'], G['random_tgt']
    thr = list(G['thresholds'])
    whole = MR.segment_rows(p, t, [0, 64], thr)
    parts = MR.segment_rows(p, t, [0, 10, 10, 40, 64], thr)
    assert np.all(parts[1] == 0)
    assert np.array_equal(parts[:, 3 + 17:].sum(0), whole[0, 3 + 17:])
    assert np.allclose(parts.sum(0), whole[0], rtol=1e-13, atol=0)


def test_zero_root_reads_a_zeroed_copy(G):
    p, t = G['random_pred'], G['random_tgt'].copy()
    before = t.copy()
    a = MR.segment_rows(p, t, [0, 64], [50.0], zero_root=True)
    z = t.copy()
    z[:, 0] = 0
    assert np.array_equal(a, MR.segment_rows(p, z, [0, 64], [50.0]))
    assert np.array_equal(t, before)
