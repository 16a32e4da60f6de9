"""The numpy restatement of the track-records kernel (tests/recordsref.py) against the host functions it replaces:
select_tracks, center_scale, affine_pair and inverse_matrix with cv2.getAffineTransform, bit for bit, and its 6 x 6
LU against cv2.getAffineTransform itself."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import recordsref as R                                              # noqa: E402
from gast_b200 import keypoints2d as K                              # noqa: E402
from gast_b200.engine import GastError                              # noqa: E402

cv2 = pytest.importorskip('cv2')


def _grid(rng, lo, hi, n):
    return np.round(rng.uniform(lo, hi, n), 2)


def _box_sets():
    """(name, boxes (n, 4) float64, (W, H), image_size, heatmap_size): 100,000+ boxes in all"""
    rng = np.random.default_rng(11)
    out = []
    # 0.01-grid boxes, partly outside the frame
    x1, y1 = _grid(rng, -300, 1920, 30000), _grid(rng, -300, 1080, 30000)
    out.append(('grid', np.stack([x1, y1, x1 + _grid(rng, 1, 800, 30000), y1 + _grid(rng, 1, 1000, 30000)], 1),
                (1920, 1080), (288, 384), (72, 96)))
    # off-grid boxes on a portrait frame
    x1, y1 = rng.uniform(-200, 1080, 20000), rng.uniform(-200, 1920, 20000)
    out.append(('offgrid', np.stack([x1, y1, x1 + rng.uniform(0.5, 900, 20000), y1 + rng.uniform(0.5, 1500, 20000)], 1),
                (1080, 1920), (288, 384), (72, 96)))
    # tiny frames
    n = 15000
    x1, y1 = rng.uniform(-5, 12, n), rng.uniform(-5, 12, n)
    boxes = np.stack([x1, y1, x1 + rng.uniform(0.01, 9, n), y1 + rng.uniform(0.01, 9, n)], 1)
    for W, H in ((1, 1), (7, 5), (3, 16)):
        out.append(('tiny_%dx%d' % (W, H), boxes[:n // 3], (W, H), (288, 384), (72, 96)))
        boxes = boxes[n // 3:]
    # bw == aspect * bh exactly: integer boxes, aspect 9/16 (1920 x 1080) and 1/2 (1000 x 500)
    for (W, H), num, den in (((1920, 1080), 9, 16), ((1000, 500), 1, 2)):
        n = 5000
        bh = rng.integers(1, 60, n) * den
        x1, y1 = rng.integers(-100, 1500, n), rng.integers(-100, 900, n)
        out.append(('aspect_%dx%d' % (W, H), np.stack([x1, y1, x1 + bh * num // den, y1 + bh], 1).astype(np.float64),
                    (W, H), (288, 384), (72, 96)))
    # width <= 0 < height
    n = 5000
    x1, y1 = _grid(rng, 0, 1900, n), _grid(rng, 0, 1000, n)
    out.append(('flat', np.stack([x1, y1, x1 - _grid(rng, 0, 50, n), y1 + _grid(rng, 0.01, 300, n)], 1),
                (1920, 1080), (288, 384), (72, 96)))
    # centred at x = -1: no 1.25 factor
    n = 3000
    a, y1 = _grid(rng, 0.01, 200, n), _grid(rng, -50, 1000, n)
    out.append(('minus_one', np.stack([-1 - a, y1, -1 + a, y1 + _grid(rng, 1, 500, n)], 1), (1920, 1080), (288, 384),
                (72, 96)))
    # tiny boxes far out, down to a triangle whose points coincide in float32 (cv2 gives a zero matrix)
    n = 4000
    x1, y1 = _grid(rng, -1e5, 1e5, n), _grid(rng, -1e5, 1e5, n)
    d = rng.choice([0.0, 0.01, 0.02, 0.05], (n, 2))
    d[d.sum(1) == 0, 1] = 0.01
    out.append(('tiny_boxes', np.stack([x1, y1, x1 + d[:, 0], y1 + d[:, 1]], 1), (1920, 1080), (288, 384), (72, 96)))
    # other crop and heatmap sizes
    x1, y1 = _grid(rng, -300, 1280, 20000), _grid(rng, -300, 720, 20000)
    boxes = np.stack([x1, y1, x1 + _grid(rng, 1, 500, 20000), y1 + _grid(rng, 1, 700, 20000)], 1)
    for k, (img, hm) in enumerate((((192, 256), (48, 64)), ((256, 256), (64, 64)), ((101, 77), (25, 19)),
                                   ((7, 1), (1, 3)))):
        out.append(('sizes_%dx%d' % img, boxes[k * 5000:(k + 1) * 5000], (1280, 720), img, hm))
    # both sides non-positive: refused
    n = 2000
    x1, y1 = _grid(rng, 0, 1900, n), _grid(rng, 0, 1000, n)
    out.append(('empty', np.stack([x1, y1, x1 - _grid(rng, 0, 50, n), y1 - _grid(rng, 0, 50, n)], 1), (1920, 1080),
                (288, 384), (72, 96)))
    return out


def test_restatement_equals_the_host_functions():
    total = zeros = 0
    for name, boxes, (W, H), img, hm in _box_sets():
        rb = R.round2(boxes)
        c, s, fwd, inv, bits = R.box_matrices(rb, H, W, img, hm)
        for i in range(len(boxes)):
            sel = K.select_tracks(boxes[i:i + 1], 1)
            assert sel[0].tobytes() == rb[i].tobytes(), (name, i)
            if bits[i]:
                want = 'not finite' if bits[i] == R.ST_NONFINITE else 'non-positive width and height'
                with pytest.raises(GastError, match=want):
                    K.center_scale(sel[0], H, W)
                continue
            hc, hs = K.center_scale(sel[0], H, W)
            hf, hi = K.affine_pair(hc, hs, img, hm)
            assert hc.tobytes() == c[i].tobytes() and hs.tobytes() == s[i].tobytes(), (name, i)
            assert hf.tobytes() == fwd[i].tobytes(), (name, i, hf, fwd[i])
            assert hi.tobytes() == inv[i].tobytes() == K.inverse_matrix(hc, hs, hm).tobytes(), (name, i)
            zeros += not hf.any()
            total += 1
        if name == 'empty':
            assert (bits == R.ST_EMPTY).all()
        if name == 'minus_one':
            assert (c[:, 0] == -1).all()
    assert total >= 100000 and zeros > 0, (total, zeros)


def test_lu_equals_cv2_on_generic_and_near_singular_triangles():
    rng = np.random.default_rng(5)
    n = 20000
    tri = [rng.normal(0, 500, (n, 2, 3, 2)).astype(np.float32)]
    # near-collinear: the third point on the line through the first two, nudged by a few ulps or less
    p = rng.normal(0, 300, (n, 2, 2, 2)).astype(np.float32)
    t = rng.uniform(-2, 2, (n, 2, 1, 1))
    third = (p[:, :, :1] + t * (p[:, :, 1:] - p[:, :, :1])).astype(np.float32)
    third = third * (1 + rng.choice([0, 1e-7, -1e-7, 1e-6], (n, 2, 1, 1))).astype(np.float32)
    tri.append(np.concatenate([p, third], 2))
    # repeated points, tiny triangles and huge offsets
    q = rng.normal(0, 1e-6, (n, 2, 3, 2)).astype(np.float32) + rng.normal(0, 1e4, (n, 2, 1, 2)).astype(np.float32)
    q[: n // 4, :, 2] = q[: n // 4, :, 0]
    tri.append(q)
    zeros = 0
    for a in tri:
        got = R.affine(a[:, 0], a[:, 1])
        for i in range(n):
            want = cv2.getAffineTransform(a[i, 0], a[i, 1])
            assert want.tobytes() == got[i].tobytes(), (i, a[i], want, got[i])
            zeros += not want.any()
    assert zeros > n // 4


def _host_records(rows, counts, num_person, W, H, img, hm):
    """the host path over one sequence: select_tracks per frame, then center_scale and the matrices per box"""
    frame, slot, fwd, inv, t_out = [], [], [], [], 0
    for t in range(len(counts)):
        k = int(counts[t])
        sel = K.select_tracks(None if k < 0 else rows[t, :k], num_person)
        if sel is None:
            continue
        for p, box in enumerate(sel[:num_person]):
            c, s = K.center_scale(box, H, W)
            f, i = K.affine_pair(c, s, img, hm)
            frame.append(t), slot.append(t_out * num_person + p), fwd.append(f), inv.append(i)
        t_out += 1
    return frame, slot, fwd, inv, t_out


@pytest.mark.parametrize('num_person', [1, 2, 3])
def test_record_rule_equals_the_host_path(num_person):
    rng = np.random.default_rng(num_person)
    K_, cap, W, H = 200, 6, 1920, 1080
    counts = rng.choice([-1, 0, 1, 2, 3, 4, 6], K_).astype(np.int32)
    if num_person == 3:
        counts[counts == 2] = 3                      # no frame the host path refuses
    x1, y1 = rng.uniform(0, 1800, (K_, cap)), rng.uniform(0, 900, (K_, cap))
    rows = np.stack([x1, y1, x1 + rng.uniform(1, 300, (K_, cap)), y1 + rng.uniform(1, 400, (K_, cap)),
                     np.tile(np.arange(1, cap + 1.0), (K_, 1))], -1)
    ref = R.track_records(rows[None], counts[None], [0], num_person, (W, H), (288, 384), (72, 96))
    frame, slot, fwd, inv, t_out = _host_records(rows, counts, num_person, W, H, (288, 384), (72, 96))
    assert list(ref['frame']) == frame and list(ref['slot']) == slot
    assert ref['forward'].tobytes() == np.asarray(fwd).tobytes() and ref['inverse'].tobytes() == np.asarray(inv).tobytes()
    assert list(ref['summary'][0]) == [len(frame), t_out, 0, -1]


def test_status_bits_and_first_frame():
    cap, W, H = 4, 640, 480
    rows = np.tile(np.array([10.0, 20.0, 110.0, 220.0, 1.0]), (5, cap, 1))
    counts = np.array([1, 2, 2, 1, 0], np.int32)
    ref = R.track_records(rows[None], counts[None], [0], 3, (W, H), (288, 384))
    assert list(ref['summary'][0]) == [2, 2, R.ST_TRACKS, 1]
    with pytest.raises(GastError, match='2 tracks in a frame for num_person = 3'):
        K.select_tracks(rows[1, :2], 3)
    rows[3, 0, 2] = np.nan
    rows[0, 0, 2:4] = rows[0, 0, :2] - 1
    ref = R.track_records(rows[None], counts[None], [4], 2, (W, H), (288, 384))
    assert list(ref['summary'][0]) == [6, 4, 4 | R.ST_NONFINITE | R.ST_EMPTY | R.ST_MATRIX, 0]
    counts = np.array([1, 5, -2], np.int32)
    ref = R.track_records(rows[None, :3], counts[None], [0], 1, (W, H), (288, 384))
    assert list(ref['summary'][0]) == [1, 1, R.ST_TRACKS | R.ST_EMPTY, 0]
