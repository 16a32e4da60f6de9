"""The person detector's letterbox and post-processing on the device (gast_b200.detection, csrc/detect.cuh) against
the reference's outputs (tests/golden/detection.npz) and the numpy restatement (tests/detectionref.py), bit for bit."""
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

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def gold():
    return load_golden('detection')


def bits_equal(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, np.float32)
    b = b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def test_letterbox_equals_the_reference(gold):
    """every golden frame size (downscales, portrait, an upscale, 7 x 5), BGR and RGB frames, numpy and CUDA"""
    m = gold['meta']
    for k, (W, H) in enumerate(m['sizes']):
        frame = R.synth_frames(1, H, W, seed=k)
        want = gold['prep_off_%d' % k].astype(np.float32) / np.float32(255)
        out = Dt.letterbox(torch.from_numpy(frame).cuda(), m['D'])
        assert out.shape == (1, 3, m['D'], m['D']) and bits_equal(out[0], want), (W, H)
        rgb = Dt.letterbox(np.ascontiguousarray(frame[..., ::-1]), m['D'], rgb_input=True)
        assert torch.equal(rgb, out)
        ipp = gold['prep_off_%d' % k].astype(np.int16) + gold['prep_ipp_diff_%d' % k]
        got = torch.round(out[0] * 255).to(torch.int16).cpu().numpy()
        assert np.abs(got - ipp).max() <= 1


@pytest.mark.parametrize('D', [160, 320, 416, 608])
def test_letterbox_equals_the_restatement(D):
    for seed, (W, H) in enumerate([(1920, 1080), (1080, 1920), (333, 1000), (2000, 37), (64, 48)]):
        frames = R.synth_frames(2, H, W, seed=seed + 3)
        out = Dt.letterbox(frames, D)
        assert bits_equal(out, R.letterbox(frames, D)), (D, W, H)


def test_person_boxes_equal_the_reference(gold):
    """none passing, no person, a single survivor, IoU either side of 0.4, the clamp, NaN objectness, several D"""
    m = gold['meta']
    for name, (D, p, nms, (W, H)) in R.prediction_sets().items():
        s = m['sets'][name]
        boxes, scores, counts = Dt.person_boxes(torch.from_numpy(p[None]).cuda(), (W, H), D, m['conf'], nms)
        n = int(counts[0])
        assert n == s['n'], name
        if n:
            assert bits_equal(boxes[0, :n], gold['det_%s_boxes' % name]), name
            assert bits_equal(scores[0, :n], gold['det_%s_scores' % name][:, 0]), name
        assert not boxes[0, n:].any() and not scores[0, n:].any()


@pytest.mark.parametrize('ties', [False, True])
def test_person_boxes_equal_the_restatement(ties):
    """many frames in one call: realistic candidate counts, exact objectness ties (lower index first), overflow of
    max_det, and every row passing"""
    D = 416
    preds = [R.many_candidates(D, n, seed=n, ties=ties) for n in (5, 17, 50, 120)]
    pred = np.stack(preds)
    sizes = [(1920, 1080), (1080, 1920), (641, 481), (7, 5)]
    boxes, scores, counts = Dt.person_boxes(torch.from_numpy(pred).cuda(), sizes, D, 0.7, 0.4, max_det=40)
    eb, es, ec, _, _ = R.person_boxes(pred, sizes, D, 0.7, 0.4, max_det=40)
    assert np.array_equal(counts.cpu().numpy(), ec)
    assert bits_equal(boxes, eb) and bits_equal(scores, es)
    # every row a person candidate (at D = 160, 1,575 rows), with ties on a coarse grid or without
    allpass = R.background(160, 9)
    allpass[:, 4] = 0.75 + 0.2 * (np.arange(allpass.shape[0]) % 7 == 0) if ties else 0.71 + 0.28 * allpass[:, 4]
    allpass[:, 5] = 0.9
    b1, s1, c1 = Dt.person_boxes(allpass[None], (1280, 720), 160, 0.7, 0.4, max_det=40)
    e1, f1, g1, _, _ = R.person_boxes(allpass[None], [(1280, 720)], 160, 0.7, 0.4, max_det=40)
    assert int(c1[0]) == g1[0] and bits_equal(b1, e1) and bits_equal(s1, f1)
    rb, rs, rc, mc, pr = Dt.person_boxes(pred, sizes, D, 0.7, 0.4, max_det=40, raw=True, extras=True)
    eb, es, ec, emc, epr = R.person_boxes(pred, sizes, D, 0.7, 0.4, max_det=40, raw=True)
    assert bits_equal(rb, eb) and bits_equal(rs, es) and bits_equal(mc, emc)
    assert np.array_equal(pr.cpu().numpy(), epr)


def test_drop_ins_match_the_goldens(gold):
    from device.lib.detector import yolo_human_det
    from device.lib.detector.yolov3.preprocess import prep_image
    from device.lib.detector.yolov3.util import write_results
    m = gold['meta']
    for k, (W, H) in enumerate(m['sizes'][:3]):
        frame = R.synth_frames(1, H, W, seed=k)[0]
        img, orig, dim = prep_image(frame, m['D'])
        assert img.is_cuda and orig is frame and dim == (W, H)
        assert bits_equal(img[0], gold['prep_off_%d' % k].astype(np.float32) / np.float32(255))
    for name, (D, p, nms, (W, H)) in R.prediction_sets().items():
        model = lambda x, cuda: torch.from_numpy(p[None]).cuda()  # noqa: E731
        b, s = yolo_human_det(np.zeros((H, W, 3), np.uint8), model, reso=D, confidence=m['conf'], nms_thresh=nms)
        if m['sets'][name]['n'] == 0:
            assert b is None and s is None, name
        else:
            assert isinstance(b, np.ndarray) and b.dtype == np.float32 and s.shape == (b.shape[0], 1)
            assert bits_equal(b, gold['det_%s_boxes' % name]) and bits_equal(s, gold['det_%s_scores' % name]), name
    sets = R.prediction_sets()
    for key, names in m['batches'].items():
        pred = torch.from_numpy(np.stack([sets[n][1] for n in names])).cuda()
        r = write_results(pred, m['conf'], 80, nms=True, nms_conf=0.4, det_hm=True)
        assert r.is_cuda and bits_equal(r, gold[key]), key
    with pytest.raises(GastError):
        write_results(pred, m['conf'], 80, nms=True, nms_conf=0.4, det_hm=False)


class _StandInDarknet:
    """a stand-in for Darknet: (T, 3, D, D) -> (T, N, 85) fixed predictions per frame, chosen by the mean of the
    frame's letterboxed input, so the predictions depend on the frame alone"""

    def __init__(self, preds):
        self.preds = torch.from_numpy(np.stack(preds)).cuda()
        self.calls = 0

    def __call__(self, x, cuda):
        self.calls += 1
        key = (x.mean(dim=(1, 2, 3)) * 1000).long() % self.preds.shape[0]
        return self.preds[key]


class _Recorder:
    """a stub tracker: records what update() receives and returns it with an id column"""

    def __init__(self):
        self.seen = []

    def update(self, dets):
        self.seen.append(np.array(dets, copy=True))
        return np.concatenate([dets.astype(np.float64), np.arange(1, len(dets) + 1)[:, None]], 1)


def _clip():
    D = 416
    sets = R.prediction_sets()
    preds = [sets['iou_edge'][1], sets['none'][1], sets['clamp'][1], sets['single'][1], sets['nan'][1]]
    frames = R.synth_frames(6, 270, 480, seed=4)
    return D, preds, frames


def _expected(frames, net, D):
    T, H, W = frames.shape[:3]
    x = torch.from_numpy(R.letterbox(frames, D)).cuda()
    pred = net(x, True).cpu().numpy()
    net.calls -= 1
    eb, _, ec, _, _ = R.person_boxes(pred, [(W, H)] * T, D, 0.7, 0.4, max_det=100)
    return [eb[t, :ec[t]] if ec[t] and eb[t, :ec[t]].any() else None for t in range(T)]


def test_video_boxes_feed_the_tracker_and_chain_into_video_keypoints():
    from gast_b200 import keypoints2d as K
    D, preds, frames = _clip()
    net = _StandInDarknet(preds)
    tracker = _Recorder()
    out = Dt.video_boxes(torch.from_numpy(frames).cuda(), net, tracker, D)
    assert net.calls == 1 and len(out) == len(frames)
    want = _expected(frames, net, D)
    fed = [w for w in want if w is not None]
    assert len(tracker.seen) == len(fed) >= 2 and any(w is None for w in want)
    for a, b in zip(tracker.seen, fed):
        assert a.dtype == np.float32 and bits_equal(a, b)
    assert [o is None for o in out] == [w is None for w in want]
    # the same frames as numpy and as RGB
    t2, t3 = _Recorder(), _Recorder()
    Dt.video_boxes(frames, net, t2, D)
    Dt.video_boxes(np.ascontiguousarray(frames[..., ::-1]), net, t3, D, rgb_input=True)
    assert all(np.array_equal(a, b) and np.array_equal(a, c) for a, b, c in zip(tracker.seen, t2.seen, t3.seen))

    class _Pose(torch.nn.Module):
        def forward(self, x):
            return torch.nn.functional.avg_pool2d(x, 4)[:, :1].repeat(1, 17, 1, 1)

    kp, sc = K.video_keypoints(frames, out, _Pose(), 1)
    assert kp.shape == (1, len(fed), 17, 2) and kp.is_cuda
    with pytest.raises(GastError):
        Dt.video_boxes(frames, net, _Recorder(), D, max_det=1)


def test_split_and_repeated_calls_give_the_same_bytes():
    D = 416
    frames = R.synth_frames(5, 300, 500, seed=8)
    whole = Dt.letterbox(frames, D)
    assert torch.equal(torch.cat([Dt.letterbox(frames[:2], D), Dt.letterbox(frames[2:], D)]), whole)
    assert torch.equal(Dt.letterbox(frames, D), whole)
    pred = torch.from_numpy(np.stack([R.many_candidates(D, n, seed=n, ties=True) for n in (8, 30, 60, 90)])).cuda()
    sizes = [(500, 300)] * 4
    b, s, c = Dt.person_boxes(pred, sizes, D)
    b1, s1, c1 = Dt.person_boxes(pred[:1], sizes[:1], D)
    b2, s2, c2 = Dt.person_boxes(pred[1:], sizes[1:], D)
    assert torch.equal(torch.cat([b1, b2]), b) and torch.equal(torch.cat([s1, s2]), s) and torch.equal(torch.cat([c1, c2]), c)
    for _ in range(3):
        bb, ss, cc = Dt.person_boxes(pred, sizes, D)
        assert torch.equal(bb, b) and torch.equal(ss, s) and torch.equal(cc, c)


def test_no_host_synchronisation():
    D = 416
    frames = torch.from_numpy(R.synth_frames(3, 300, 500, seed=8)).cuda()
    pred = torch.from_numpy(np.stack([R.many_candidates(D, n, seed=n) for n in (8, 30, 60)])).cuda()
    sizes = torch.tensor([[500, 300]] * 3, dtype=torch.int32).cuda()
    Dt.letterbox(frames, D)
    Dt.person_boxes(pred, sizes, D)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        x = Dt.letterbox(frames, D)
        b, s, c = Dt.person_boxes(pred, sizes, D)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert x.shape == (3, 3, D, D) and b.shape == (3, 100, 4)


def test_refusals_before_launch():
    with pytest.raises(GastError):
        Dt.letterbox(np.zeros((1, 5, 5, 3), np.uint8), 400)
    with pytest.raises(GastError):
        Dt.person_boxes(torch.zeros((1, 10647, 84), device='cuda'), (10, 10), 416)
    with pytest.raises(GastError):
        Dt.person_boxes(torch.zeros((1, 10646, 85), device='cuda'), (10, 10), 416)
    with pytest.raises(GastError):
        Dt.person_boxes(torch.zeros((1, R.num_predictions(672), 85), device='cuda'), (10, 10), 672)
