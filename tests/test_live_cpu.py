"""The numpy restatement of the live tick's kernels (tests/liveref.py) against the host functions it restates: the
slot geometry against select_tracks without its rounding, center_scale, affine_pair and inverse_matrix with cv2, bit
for bit; the slot rule on hand-built id sequences; the inputs and the placement against tests/preprocessref.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import liveref as LR                                                # noqa: E402
import preprocessref as PR                                          # noqa: E402
from gast_b200 import keypoints2d as K                              # noqa: E402

F32 = np.float32


def _boxes():
    """(boxes (n, 4) float64, (W, H)): the §8.9 families on 0.01 grids and unrounded off-grid rows"""
    rng = np.random.default_rng(3)
    out = []
    x1, y1 = np.round(rng.uniform(-300, 1920, 4000), 2), np.round(rng.uniform(-300, 1080, 4000), 2)
    out.append((np.stack([x1, y1, x1 + np.round(rng.uniform(1, 800, 4000), 2),
                          y1 + np.round(rng.uniform(1, 1000, 4000), 2)], 1), (1920, 1080)))
    x1, y1 = rng.uniform(-200, 1080, 4000), rng.uniform(-200, 1920, 4000)
    out.append((np.stack([x1, y1, x1 + rng.uniform(0.5, 900, 4000), y1 + rng.uniform(0.5, 1500, 4000)], 1),
                (1080, 1920)))
    x1 = rng.uniform(0, 500, 500)
    out.append((np.stack([x1, x1, x1 + 320, x1 + 180], 1), (640, 360)))            # exact-aspect boxes
    out.append((np.stack([x1, x1, x1 + 50, x1], 1), (640, 360)))                    # flat boxes
    out.append((np.stack([-1 - x1, x1, -1 + x1, x1 + 9], 1), (640, 360)))           # centred at x = -1
    out.append((np.array([[5.0, 5.0, 5.0, 5.0], [7.0, 7.0, 3.0, 3.0], [np.nan, 1, 2, 3], [0, np.inf, 2, 3]]),
                (640, 360)))
    return out


def test_slot_geometry_equals_the_host_functions_without_rounding():
    pytest.importorskip('cv2')
    for boxes, (W, H) in _boxes():
        c, s, fwd, inv, bits = LR.slot_geometry(boxes, H, W, K.IMAGE_SIZE, (72, 96))
        for i, box in enumerate(boxes):
            try:
                hc, hs = K.center_scale(box, H, W)
                hf, _ = K.affine_pair(hc, hs, K.IMAGE_SIZE)
                hi = K.inverse_matrix(hc, hs, (72, 96))
            except K.GastError:
                assert bits[i] & (LR.ST_NONFINITE | LR.ST_EMPTY)
                assert not fwd[i].any() and not inv[i].any()
                continue
            if not np.isfinite(hf).all():
                assert bits[i] & LR.ST_MATRIX
                continue
            assert bits[i] == 0
            assert c[i].tobytes() == hc.tobytes() and s[i].tobytes() == hs.tobytes()
            assert fwd[i].tobytes() == hf.tobytes() and inv[i].tobytes() == hi.tobytes()


def test_selection_follows_gen_img_kpts():
    assert LR.select(-1, 2, 8) == ([], 0) and LR.select(0, 2, 8) == ([], 0)
    assert LR.select(1, 3, 8) == ([0], 0)
    assert LR.select(5, 2, 8) == ([4, 3], 0)
    assert LR.select(2, 3, 8) == ([], LR.ST_TRACKS)
    assert LR.select(9, 2, 8) == ([], LR.ST_TRACKS)
    # select_tracks without its round(v, 2) picks the same rows
    t = np.arange(25, dtype=np.float64).reshape(5, 5) + 0.123
    rows, _ = LR.select(5, 2, 8)
    assert np.array_equal(K.select_tracks(t, 2), np.round(t[rows, :4], 2))


def _run(book, seq):
    return [book.assign(ids, tick) for tick, ids in enumerate(seq)]


def test_slot_rule_entering_leaving_missed_and_swapping():
    b = LR.SlotBook(2)
    slots = _run(b, [[7], [7, 9], [9, 7], [9], [7, 9], [], [9, 7]])
    assert slots == [[0], [0, 1], [1, 0], [1], [0, 1], [], [1, 0]]
    assert b.ids.tolist() == [7, 9]                  # the ids kept their slots through the swap and the miss


def test_slot_rule_restarts_only_on_a_new_id():
    b = LR.SlotBook(2)
    b.assign([3], 0)
    b.fresh[:] = False
    b.assign([3, 4], 1)
    assert b.fresh.tolist() == [False, True]
    b.fresh[:] = False
    b.assign([5], 2)                                 # slot 1 seen at tick 1, slot 0 at tick 1: the lower slot goes
    assert b.ids.tolist() == [5, 4] and b.fresh.tolist() == [True, False]


def test_slot_rule_more_ids_than_slots_takes_the_oldest():
    b = LR.SlotBook(2)
    b.assign([1, 2], 0)
    b.assign([1], 1)
    assert b.assign([3], 2) == [1]                   # slot 1 (id 2) was seen longest ago
    assert b.assign([4, 1], 3) == [1, 0]
    assert b.ids.tolist() == [1, 4]
    b = LR.SlotBook(1)
    assert _run(b, [[1], [2], [2], [1]]) == [[0], [0], [0], [0]] and b.ids.tolist() == [1]


def _coco(rng, n):
    kp = rng.uniform(10, 600, (n, 17, 2)).astype(F32)
    sc = rng.uniform(0, 1, (n, 17)).astype(F32)
    kp[1] = 0                                        # absent
    kp[2, :, 0] = 0                                  # present, but a zero x sum
    sc[3, [2, 3, 5, 6]] = 0.1
    return kp, sc


def test_inputs_equal_preprocessref_on_single_frames():
    rng = np.random.default_rng(5)
    kp, sc = _coco(rng, 40)
    slot_active = rng.random(40) < 0.8
    W, H = 640, 360
    kpts, scores, x, active = LR.inputs(kp, sc, slot_active, W, H)
    for s in range(40):
        hk, hs, frames = PR.h36m_coco_format(kp[s][None, None], sc[s][None, None])
        is_active = slot_active[s] and len(frames) == 1 and frames[0].size == 1
        assert active[s] == is_active
        if not is_active:
            assert not kpts[s].any() and not scores[s].any() and not x[s].any()
            continue
        re = PR.revise_kpts(hk, hs, frames)[0, 0]
        assert kpts[s].tobytes() == re.tobytes() and scores[s].tobytes() == hs[0, 0].tobytes()
        norm = (re / F32(W) * F32(2) - np.array([1, H / W])).astype(F32)     # normalize_screen_coordinates
        assert x[s].tobytes() == norm.tobytes()


def test_place_equals_preprocessref_over_the_active_slots():
    rng = np.random.default_rng(6)
    C, P, W = 3, 2, 640
    world = rng.normal(0, 1, (C * P, 17, 3)).astype(F32)
    kpts = rng.uniform(0, 600, (C * P, 17, 2)).astype(F32)
    active = np.array([1, 0, 1, 1, 0, 0], bool)
    out = LR.place(world, kpts, active, C, P, W).reshape(C, P, 17, 3)
    for c in range(C):
        a = active.reshape(C, P)[c]
        assert not out[c, ~a].any()
        if a.any():
            ref = PR.revise_skes_real_time(world.reshape(C, P, 17, 3)[c, a], kpts.reshape(C, P, 17, 2)[c, a], W)
            assert out[c, a].tobytes() == ref.tobytes()
