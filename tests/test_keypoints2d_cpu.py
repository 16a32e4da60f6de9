"""The 2D pose net's crop and heatmap decode without a GPU: the numpy restatement (tests/keypoints2dref.py) against the
reference's outputs (tests/golden/keypoints2d.npz, made by make_golden_keypoints2d.py), the warp restatement against
live cv2.warpAffine, the host box geometry of gast_b200.keypoints2d, and the refusals."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import keypoints2dref as R                                          # noqa: E402
from conftest import load_golden                                    # noqa: E402
from gast_b200 import keypoints2d as K                              # noqa: E402
from gast_b200.engine import GastError                              # noqa: E402

try:
    import cv2
except ImportError:
    cv2 = None


@pytest.fixture(scope='module')
def gold():
    g = load_golden('keypoints2d')
    m = g['meta']
    g['frames'] = R.synth_frames(m['F'], m['H'], m['W'])
    return g


def bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def test_warp_restatement_equals_cv2_goldens(gold):
    m = gold['meta']
    for k in range(len(gold['boxes'])):
        f = gold['frames'][gold['box_frame'][k]]
        assert np.array_equal(R.warp(f, gold['fwd_small'][k], *m['small']), gold['warps_small'][k]), k
        if k < m['full_n']:
            assert np.array_equal(R.warp(f, gold['fwd_full'][k], *m['full']), gold['warps_full'][k]), k


def test_preprocess_restatement_equals_reference(gold):
    m = gold['meta']
    for i, (f, b0, nb, num_pos) in enumerate(m['pre_calls']):
        boxes = gold['boxes'][b0:b0 + min(nb, num_pos)]
        for r, box in enumerate(boxes):
            c, s = R.center_scale(box, m['H'], m['W'])
            assert bits_equal(c, gold['pre%d_centers' % i][r]) and bits_equal(s, gold['pre%d_scales' % i][r])
            crop = R.crop(gold['frames'][f], gold['pre%d_fwd' % i][r], m['pre_size'], net_order=False)
            assert bits_equal(crop, gold['pre%d_inputs' % i][r]), (i, r)
            # the net's plane order and RGB input are permutations of the same planes
            assert bits_equal(R.crop(gold['frames'][f], gold['pre%d_fwd' % i][r], m['pre_size']), crop[::-1])
            rgb = np.ascontiguousarray(gold['frames'][f][..., ::-1])
            assert bits_equal(R.crop(rgb, gold['pre%d_fwd' % i][r], m['pre_size'], rgb_input=True, net_order=False), crop)


@pytest.mark.parametrize('size', [(72, 96), (48, 64)])
@pytest.mark.parametrize('post', [True, False])
def test_decode_restatement_equals_reference(gold, size, post):
    hw, hh = size
    hm = np.concatenate([R.edge_case_heatmaps(hh, hw), R.synth_heatmaps(4, 17, hh, hw, seed=3)])
    inv = gold['inv_%dx%d' % size][:hm.shape[0]]
    p, mv = R.decode(hm, inv, post)
    key = 'dec_%dx%d_%s' % (hw, hh, 'post' if post else 'plain')
    assert bits_equal(p, gold[key + '_preds'])
    assert bits_equal(mv, gold[key + '_maxvals'])


def test_edge_cases_reach_every_branch():
    hm = R.edge_case_heatmaps(96, 72)
    p, mv = R.decode(hm, np.tile(np.array([[1., 0, 0], [0, 1., 0]]), (hm.shape[0], 1, 1)), True)
    assert np.isnan(mv[0, 3, 0]) and np.isnan(mv[0, 4, 0])          # NaN map, NaN after the peak
    assert np.all(p[0, 3] == 0) and np.all(p[0, 0] == 0)            # masked: NaN, negative
    assert np.all(np.isnan(p[0, 5]))                                # NaN difference
    assert mv[0, 6, 0] == np.inf and p[0, 6, 1] == 48.25            # inf peak, inf difference
    assert np.all(np.abs(p[0, 2] - [4.0, 3.0]) <= 0.25)            # equal peaks: the first wins
    xs = {float(v) % 1 for v in p[1:, :, 0].ravel()} | {float(v) % 1 for v in p[1:, :, 1].ravel()}
    assert {0.0, 0.25, 0.75} <= xs                                  # shifts both ways, and none at the borders


def test_host_geometry_equals_reference(gold, monkeypatch):
    """box_to_center_scale with the frame's H and W as the model size (the reference's argument order), the float32
    triangles, and the matrices: cv2's bit for bit, the closed form within a few ulps"""
    m = gold['meta']
    H, W = m['H'], m['W']
    for k, box in enumerate(gold['boxes']):
        c, s = K.center_scale([v for v in box], H, W)
        assert bits_equal(c, gold['centers'][k]) and bits_equal(s, gold['scales'][k])
        assert bits_equal(c, R.center_scale(box, H, W)[0]) and bits_equal(s, R.center_scale(box, H, W)[1])
        assert abs(s[0] / s[1] - H / W) < 1e-6                      # the H/W aspect, not 288/384
        rs, rd = R.triangles(c, s, m['full'])
        ks, kd = K.triangles(c, s, m['full'])
        assert bits_equal(rs, ks) and bits_equal(rd, kd)
    for closed in ([False, True] if cv2 is not None else [True]):
        if closed:
            monkeypatch.setattr(K, '_cv2', None)
        for k in range(len(gold['boxes'])):
            c, s = gold['centers'][k], gold['scales'][k]
            fwd, inv = K.affine_pair(c, s, m['full'], (72, 96))
            for got, want in ((fwd, gold['fwd_full'][k]), (inv, gold['inv_72x96'][k]),
                              (K.inverse_matrix(c, s, (48, 64)), gold['inv_48x64'][k])):
                if closed:
                    assert np.allclose(got, want, rtol=1e-12, atol=1e-9)
                else:
                    assert np.array_equal(got, want)


def test_select_tracks_follows_gen_video_kpts():
    rs = np.random.default_rng(3)
    tr = rs.uniform(0, 1000, (4, 5))

    def ref(t, num):                                                # gen_kpts.py:214-226
        if t.shape[0] == 1:
            kept = t[-1, :-1].reshape(1, 4)
        else:
            kept = t[-num:, :-1].reshape(num, 4)[::-1]
        return np.array([[round(i, 2) for i in list(b)] for b in kept])
    for k, num in [(1, 1), (1, 2), (4, 1), (4, 2), (3, 3), (2, 2)]:
        assert np.array_equal(K.select_tracks(tr[:k], num), ref(tr[:k], num)), (k, num)
    assert K.select_tracks(None, 2) is None and K.select_tracks(np.zeros((0, 5)), 2) is None
    with pytest.raises(GastError):
        K.select_tracks(tr[:2], 3)                                  # the reference's reshape raises
    with pytest.raises(ValueError):
        ref(tr[:2], 3)


@pytest.mark.skipif(cv2 is None, reason='cv2 is not importable')
def test_warp_restatement_equals_live_cv2():
    """hundreds of random matrices on landscape, portrait, odd-sized and tiny frames, with boxes wholly inside,
    partly outside and wholly outside"""
    rs = np.random.default_rng(11)
    n = 0
    for H, W in [(1080, 1920), (1920, 1080), (37, 53), (481, 641), (5, 7)]:
        img = rs.integers(0, 256, (H, W, 3), dtype=np.uint8)
        for t in range(80):
            s = rs.uniform(0.05, 4.0)
            a0, a4 = s * rs.choice([-1, 1]) * rs.uniform(0.7, 1.3), s * rs.choice([-1, 1])
            a1 = rs.uniform(-1, 1) * s * (t % 3 == 0)
            a3 = rs.uniform(-1, 1) * s * (t % 5 == 0)
            M = np.array([[a0, a1, rs.uniform(-2.5, 1.5) * W * s], [a3, a4, rs.uniform(-2.5, 1.5) * H * s]])
            ow, oh = [(288, 384), (13, 9), (72, 96), (48, 64)][t % 4]
            assert np.array_equal(R.warp(img, M, ow, oh), cv2.warpAffine(img, M, (ow, oh), flags=cv2.INTER_LINEAR))
            n += 1
    # the reference's own matrices: boxes partly outside a 1920 x 1080 frame
    img = rs.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    for t in range(60):
        x1, y1 = rs.uniform(-300, 1800), rs.uniform(-300, 1000)
        box = np.round([x1, y1, x1 + rs.uniform(20, 700), y1 + rs.uniform(40, 1000)], 2)
        c, s = K.center_scale(box, 1080, 1920)
        M = K.affine_pair(c, s)[0]
        assert np.array_equal(R.warp(img, M, 288, 384), cv2.warpAffine(img, M, (288, 384), flags=cv2.INTER_LINEAR))
        n += 1
    assert n == 460


def test_refusals():
    with pytest.raises(GastError):
        K.center_scale([10.0, 10.0, 10.0, 5.0], 1080, 1920)          # no width, negative height
    with pytest.raises(GastError):
        K.center_scale([10.0, np.nan, 50.0, 90.0], 1080, 1920)
    frames = np.zeros((2, 8, 8, 3), np.uint8)
    eye = np.array([[1., 0, 0], [0, 1., 0]])
    with pytest.raises(GastError):
        K.crop_persons(frames, [2], eye[None], (4, 4))              # frame index out of range
    with pytest.raises(GastError):
        K.crop_persons(frames, [0], np.array([[[1., 0, np.inf], [0, 1., 0]]]), (4, 4))
    with pytest.raises(GastError):
        K.crop_persons(np.zeros((1, 32768, 1, 3), np.uint8), [0], eye[None], (4, 4))
    with pytest.raises(GastError):
        K.crop_persons(frames, [0], eye[None], (32768, 4))
    with pytest.raises(GastError):
        K.crop_persons(frames[..., :2], [0], eye[None], (4, 4))
    with pytest.raises(GastError):
        K.decode_heatmaps(np.zeros((1, 33, 8, 8), np.float32), eye[None])
    with pytest.raises(GastError):
        K.decode_heatmaps(np.zeros((1, 17, 8, 257), np.float32), eye[None])
    with pytest.raises(GastError):
        K.decode_heatmaps(np.zeros((1, 17, 8, 8), np.float64), eye[None])
    with pytest.raises(GastError):
        K.decode_heatmaps(np.zeros((1, 17, 8, 8), np.float32), np.full((1, 2, 3), np.nan))
    with pytest.raises(GastError):
        K.video_keypoints(frames, [np.array([[0., 0, 4, 4, 1], [1., 1, 5, 5, 2]]), None], None, 3)
