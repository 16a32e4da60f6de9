"""The person detector's letterbox and post-processing without a GPU: the numpy restatement (tests/detectionref.py)
against the reference's outputs (tests/golden/detection.npz, made by make_golden_detection.py), the letterbox against
live cv2 with IPP off (exact) and on (within one grey level), round(v, 2), the tie order, and the refusals of
gast_b200.detection."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import detectionref as R                                            # noqa: E402
from conftest import load_golden                                    # noqa: E402
from gast_b200 import detection as Dt                               # noqa: E402
from gast_b200.engine import GastError                              # noqa: E402

try:
    import cv2
except ImportError:
    cv2 = None

needs_cv2 = pytest.mark.skipif(cv2 is None, reason='cv2 is not installed')


@pytest.fixture(scope='module')
def gold():
    return load_golden('detection')


def bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def test_letterbox_restatement_equals_the_goldens(gold):
    m = gold['meta']
    for k, (W, H) in enumerate(m['sizes']):
        frame = R.synth_frames(1, H, W, seed=k)
        x = R.letterbox(frame, m['D'])[0]
        assert bits_equal(x, gold['prep_off_%d' % k].astype(np.float32) / np.float32(255)), (W, H)
        ipp = gold['prep_off_%d' % k].astype(np.int16) + gold['prep_ipp_diff_%d' % k]
        assert np.abs(np.rint(x * 255).astype(np.int16) - ipp).max() <= 1


def test_letterbox_planes_are_the_reference_division():
    """u8 / 255 as torch divides: the correctly rounded float32 quotient for all 256 values"""
    v = np.arange(256, dtype=np.uint8).reshape(1, 1, 256).repeat(3, 0).transpose(1, 2, 0)
    want = torch.from_numpy(np.arange(256)).float().div(255.0).numpy()
    got = R.to_planes(v)
    assert all(bits_equal(got[c, 0], want) for c in range(3))


@needs_cv2
def test_resize_restatement_equals_cv2_without_ipp():
    """a few hundred sizes, extreme aspect ratios, down- and upscales, at several inp_dim"""
    rs = np.random.default_rng(11)
    use = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        sizes = [(1, 1), (1, 700), (700, 1), (2, 3000), (3000, 2), (7, 5), (416, 416), (417, 415), (32767, 3),
                 (3, 20000)]
        sizes += [(int(rs.integers(1, 2200)), int(rs.integers(1, 2200))) for _ in range(230)]
        for k, (W, H) in enumerate(sizes):
            D = (160, 320, 416, 608)[k % 4]
            nw, nh, _, _ = R.letterbox_geometry(W, H, D)
            if nw == 0 or nh == 0:
                continue
            img = rs.integers(0, 256, (H, W, 3), dtype=np.uint8)
            if k % 3 == 0:
                img = R.synth_frames(1, H, W, seed=k)[0]
            want = cv2.resize(img, (nw, nh), interpolation=cv2.INTER_CUBIC)
            assert np.array_equal(R.resize_cubic(img, nw, nh), want), (W, H, D)
    finally:
        cv2.ipp.setUseIPP(use)


@needs_cv2
def test_resize_restatement_within_one_level_of_cv2_with_ipp():
    rs = np.random.default_rng(12)
    use = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(True)
    try:
        for W, H in [(1920, 1080), (1080, 1920), (1280, 720), (641, 481), (320, 240), (97, 2000)]:
            img = rs.integers(0, 256, (H, W, 3), dtype=np.uint8)
            nw, nh, _, _ = R.letterbox_geometry(W, H, 416)
            want = cv2.resize(img, (nw, nh), interpolation=cv2.INTER_CUBIC).astype(np.int16)
            assert np.abs(R.resize_cubic(img, nw, nh).astype(np.int16) - want).max() <= 1
    finally:
        cv2.ipp.setUseIPP(use)


def test_person_boxes_restatement_equals_the_goldens(gold):
    m = gold['meta']
    for name, (D, p, nms, (W, H)) in R.prediction_sets().items():
        boxes, scores, counts, _, _ = R.person_boxes(p[None], [(W, H)], D, m['conf'], nms)
        n = int(counts[0])
        assert n == m['sets'][name]['n'], name
        if n:
            assert bits_equal(boxes[0, :n], gold['det_%s_boxes' % name]), name
            assert bits_equal(scores[0, :n], gold['det_%s_scores' % name][:, 0]), name


def test_write_results_restatement_equals_the_goldens(gold):
    """the raw corners, objectness and class-score columns of a two-image batch, and the early return"""
    m = gold['meta']
    sets = R.prediction_sets()
    names = m['batches']['wr_two']
    pred = np.stack([sets[n][1] for n in names])
    b, s, c, mc, _ = R.person_boxes(pred, [(416, 416)] * 2, 416, m['conf'], 0.4, max_det=50, raw=True)
    rows = np.concatenate([np.concatenate([np.full((c[i], 1), i, np.float32), b[i, :c[i]], s[i, :c[i], None],
                                           mc[i, :c[i], None], np.zeros((c[i], 1), np.float32)], 1) for i in range(2)])
    assert bits_equal(rows, gold['wr_two'])
    names = m['batches']['wr_early']
    pred = np.stack([sets[n][1] for n in names])
    _, _, _, _, persons = R.person_boxes(pred, [(416, 416)] * 3, 416, m['conf'], 0.4, raw=True)
    assert persons[1] == 0 and gold['wr_early'].shape == (0, 7)


def test_round2_is_numpys_round_over_a_wide_range():
    rs = np.random.default_rng(3)
    v = np.concatenate([rs.uniform(-5000, 5000, 200000), rs.uniform(-1, 1, 50000),
                        np.arange(-200000, 200000) / 100.0 + 0.005, [0.0, -0.0, 1e6, 3e7, 1e-30]]).astype(np.float32)
    want = np.array([round(x, 2) for x in v], np.float32)
    assert bits_equal(R.round2(v), want)
    bits = rs.integers(0, 0x7f800000, 100000, dtype=np.int64).astype(np.uint32).view(np.float32)
    bits = bits[np.abs(bits) < 3e38]
    assert bits_equal(R.round2(bits), np.array([round(x, 2) for x in bits], np.float32))


def test_scale_factor_is_torchs_reciprocal_product():
    """torch.min(inp_dim / img_dim, 1): a python int over a float32 tensor"""
    rs = np.random.default_rng(4)
    for W, H in [(1920, 1080), (1080, 1920), (7, 5), (641, 481)] + [tuple(rs.integers(1, 5000, 2)) for _ in range(3000)]:
        for D in (160, 416, 608):
            t = torch.FloatTensor([W, H]).repeat(1, 2)
            want = torch.min(D / t, 1)[0].item()
            assert np.float32(want) == R.scale_factor(D, W, H), (W, H, D)


def test_ties_keep_the_lower_index_first():
    D = 416
    p = R.background(D, 21)
    for r, obj in ((900, 1.0), (50, 1.0), (4000, 0.9), (20, 0.9), (10000, np.nan), (7, np.nan)):
        R.put(p, r, 30 + (r % 300), 40 + (r % 200), 10.0, 10.0, obj)
        p[r, 5] = np.nan if np.isnan(obj) else p[r, 5]
    cands, _ = R.candidates(p, 0.7)
    rows = [r[0] for r in R.nms(cands, 0.4)]
    assert rows == [7, 10000, 50, 900, 20, 4000]


def test_refusals():
    with pytest.raises(GastError):
        Dt.letterbox(np.zeros((1, 5, 5, 3), np.float32), 416)
    with pytest.raises(GastError):
        Dt.letterbox(np.zeros((1, 5, 5), np.uint8), 416)
    with pytest.raises(GastError):
        Dt.letterbox(np.zeros((1, 5, 32768, 3), np.uint8), 416)
    with pytest.raises(GastError):
        Dt.letterbox(np.zeros((1, 1, 2000, 3), np.uint8), 416)        # new_h = int(1 * 0.208) = 0
    for D in (32, 400, 0):
        with pytest.raises(GastError):
            Dt.letterbox(np.zeros((1, 5, 5, 3), np.uint8), D)
        with pytest.raises(GastError):
            Dt.check_inp_dim(D)
    with pytest.raises(GastError):
        Dt.check_inp_dim(672)                                           # 27783 predictions: beyond one CTA
    assert Dt.check_inp_dim(640) == 640
    with pytest.raises(GastError):
        Dt.person_boxes(np.zeros((1, 10647, 85), np.float64), (10, 10), 416)
    with pytest.raises(GastError):
        Dt.person_boxes(np.zeros((1, 10647, 84), np.float32), (10, 10), 416)
    with pytest.raises(GastError):
        Dt.person_boxes(np.zeros((1, 10646, 85), np.float32), (10, 10), 416)
    with pytest.raises(GastError):
        Dt.person_boxes(np.zeros((1, 10647, 85), np.float32), (10, 10), 416, max_det=-1)
    assert Dt.num_predictions(416) == 10647 and Dt.num_predictions(608) == 22743
    from device.lib.detector.yolov3.util import write_results
    with pytest.raises(GastError):
        write_results(torch.zeros((1, 10647, 85)), 0.7, 80, det_hm=False)
