"""SORT on the device (gast_b200.tracking, csrc/track.cuh) against the reference's outputs (tests/golden/sort.npz)
and the numpy restatement (tests/sortref.py): counts, ids and row order exactly, boxes within 1e-12 of each box's
largest coordinate (S^-1 and the Kalman-gain products are fp64 in an order of their own)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sortref as R                                                 # noqa: E402
from conftest import load_golden                                    # noqa: E402
from gast_b200 import tracking as Tk                                # noqa: E402
from gast_b200.engine import GastError                              # noqa: E402

pytestmark = pytest.mark.gpu
BOX_TOL = 1e-12
HALF_TOL = 1e-9
NEAR_HALF = []          # (where, value) of boxes within HALF_TOL of a round(v, 2) half, reported at the end


def _close(got, want, where):
    """one frame's rows: same count, ids and order; boxes within BOX_TOL of the box's largest coordinate and equal
    after round(v, 2) unless the value sits within HALF_TOL of a rounding half"""
    assert got.shape == want.shape, (where, got.shape, want.shape)
    assert np.array_equal(got[:, 4], want[:, 4]), (where, got[:, 4], want[:, 4])
    g, w = got[:, :4], want[:, :4]
    nan = np.isnan(w)
    assert np.array_equal(np.isnan(g), nan), where
    scale = np.maximum(np.nanmax(np.abs(np.where(nan, 0, w)), axis=1, keepdims=True), 1.0)
    err = np.abs(np.where(nan, 0, g - w))
    assert (err <= BOX_TOL * scale).all(), (where, float((err / scale).max()))
    half = np.abs(np.where(nan, 0, w) * 100 - np.floor(np.where(nan, 0, w) * 100) - 0.5) < HALF_TOL * 100
    for v in w[half]:
        NEAR_HALF.append((where, float(v)))
    ok = half | nan | (np.round(np.where(nan, 0, g), 2) == np.round(np.where(nan, 0, w), 2))
    assert ok.all(), where


def _same_lists(got, want, where):
    assert len(got) == len(want), where
    for t, (a, b) in enumerate(zip(got, want)):
        assert (a is None) == (b is None), (where, t)
        if a is not None:
            _close(a, np.asarray(b).reshape(-1, 5), (where, t))


def _device_run(frames, max_age, min_hits, skip_empty=False, chunks=None, capacity=256):
    trk = Tk.DeviceSort(1, max_age, min_hits, capacity)
    boxes, counts = R.pack(frames)
    out, t0 = [], 0
    for k in (chunks or [len(frames)]):
        out += Tk.host_tracks(*trk.update_chunk(boxes[t0:t0 + k], counts[t0:t0 + k], skip_empty))
        t0 += k
    return out


def _bits(lists):
    return [None if a is None else a.tobytes() for a in lists]


@pytest.fixture(scope='module')
def gold():
    return load_golden('sort')


def test_goldens(gold):
    meta = gold['meta']['scenarios']
    for name, (max_age, min_hits, frames) in R.scenarios().items():
        m = meta[name]
        stop = m['raised']['frame'] if m['raised'] else len(frames)
        out = _device_run(frames[:stop], max_age, min_hits)
        counts = gold['%s_counts' % name]
        assert [len(o) for o in out] == list(counts), name
        rows = gold['%s_rows' % name]
        at = np.concatenate([[0], np.cumsum(counts)])
        for t, o in enumerate(out):
            _close(o, rows[at[t]:at[t + 1]], (name, t))
        if m['raised']:
            trk = Tk.DeviceSort(1, max_age, min_hits)
            b, n = R.pack(frames)
            with pytest.raises(GastError, match='IoU'):
                Tk.host_tracks(*trk.update_chunk(b, n, skip_empty=False))


def test_random_sequences_against_the_restatement():
    """20,000 frames: 4 sequences of 5,000 with 0 - 12 persons, clutter and dropouts, in one launch; each sequence alone
    gives the same bits"""
    seqs = [R.random_sequence(5000, seed) for seed in range(4)]
    M = max(len(f) for s in seqs for f in s)
    packed = [R.pack(s, M) for s in seqs]
    boxes = np.stack([p[0] for p in packed])
    counts = np.stack([p[1] for p in packed])
    trk = Tk.DeviceSort(4, 1, 3)
    got = Tk.host_tracks(*trk.update_chunk(boxes, counts, skip_empty=False))
    for s, frames in enumerate(seqs):
        _same_lists(got[s], R.run(frames, 1, 3), ('random', s))
        alone = Tk.DeviceSort(1, 1, 3)
        one = Tk.host_tracks(*alone.update_chunk(boxes[s], counts[s], skip_empty=False))
        assert _bits(one) == _bits(got[s]), s
    print('\nrandom sequences: %d rows, %d persons at most per frame' % (
        sum(len(o) for g in got for o in g), M))


def test_chunking_and_repeats_give_the_same_bits():
    frames = R.random_sequence(600, 11)
    whole = _device_run(frames, 1, 3)
    assert _bits(_device_run(frames[:300], 1, 3, chunks=[1] * 300)) == _bits(whole[:300])
    assert _bits(_device_run(frames, 1, 3, chunks=[1, 7, 100, 292, 200])) == _bits(whole)
    for _ in range(2):
        assert _bits(_device_run(frames, 1, 3)) == _bits(whole)


def test_skip_empty():
    frames = R.random_sequence(300, 5)
    for t in range(0, 300, 17):
        frames[t] = np.zeros((0, 4), np.float32)
    for t in range(5, 300, 29):
        frames[t] = np.zeros((2, 4), np.float32)           # boxes that are all zero
    on = _device_run(frames, 1, 3, skip_empty=True)
    want = R.run(frames, 1, 3, skip_empty=True)
    assert sum(o is None for o in on) == sum(w is None for w in want) > 20
    _same_lists(on, want, 'skip')
    off = _device_run(frames, 1, 3, skip_empty=False)
    _same_lists(off, R.run(frames, 1, 3), 'noskip')
    assert all(o is not None for o in off)


class _Restated:
    def __init__(self):
        self.s = R.Sort()

    def update(self, dets):
        return self.s.update(dets)


def test_video_boxes_with_device_sort_chain_into_video_keypoints():
    import detectionref as DR
    from gast_b200 import detection as Dt
    from gast_b200 import keypoints2d as K
    sets = DR.prediction_sets()
    preds = [sets[k][1] for k in ('iou_edge', 'none', 'clamp', 'single', 'nan')]
    frames = DR.synth_frames(12, 270, 480, seed=4)

    class Net:
        def __init__(self):
            self.p = torch.from_numpy(np.stack(preds)).cuda()

        def __call__(self, x, cuda):
            return self.p[(x.mean(dim=(1, 2, 3)) * 1000).long() % self.p.shape[0]]

    dev = Dt.video_boxes(torch.from_numpy(frames).cuda(), Net(), Tk.DeviceSort(), 416)
    host = Dt.video_boxes(frames, Net(), _Restated(), 416)
    assert any(o is None for o in host) and any(o is not None and len(o) for o in host)
    _same_lists(dev, host, 'video_boxes')

    class Pose(torch.nn.Module):
        def forward(self, x):
            return torch.nn.functional.avg_pool2d(x, 4)[:, :1].repeat(1, 17, 1, 1)

    kp, sc = K.video_keypoints(frames, dev, Pose(), 1)
    assert kp.is_cuda and kp.shape[-2:] == (17, 2)


def test_drop_in_sort_numbers_ids_across_instances():
    from device.lib.track import sort as S
    S.KalmanBoxTracker.count = 0
    a_frames, b_frames = R.random_sequence(120, 21, 5), R.random_sequence(120, 22, 5)
    a, b = S.Sort(), S.Sort(max_age=2, min_hits=1)
    ra, rb = R.Sort(), R.Sort(max_age=2, min_hits=1)
    count = 0
    for t in range(120):
        for dev, ref, fr in ((a, ra, a_frames[t]), (b, rb, b_frames[t])):
            dets = np.concatenate([fr, np.ones((len(fr), 1), np.float32)], 1) if t % 2 else fr
            ref.next_id = count
            want = ref.update(dets)
            count = ref.next_id
            got = dev.update(dets)
            assert got.dtype == np.float64
            _close(got, want, ('drop-in', t))
    assert S.KalmanBoxTracker.count == count > 20
    with pytest.raises(GastError):
        a.update(R._boxes([[0, 0, 100, 100]]).astype(np.float64))


def _header_offsets(cap):
    a = lambda o: (o + 15) // 16 * 16                     # noqa: E731
    o = 64
    for size in (4, 4, 4, 4, 4, 4, 8):
        o = a(o + cap * size)
    return o                                              # start of x[cap][8]


def test_status_words_raise():
    one = R._boxes([[10000, 10000, 15000, 20000]])
    b, n = R.pack([one, one])
    # a count above max_det
    trk = Tk.DeviceSort()
    with pytest.raises(GastError, match='max_det'):
        Tk.host_tracks(*trk.update_chunk(b, np.array([1, 2], np.int32)))
    with pytest.raises(GastError, match='max_det'):         # the word stays set
        Tk.host_tracks(*trk.update_chunk(b, n))
    # a tracker list beyond its capacity
    three = R._boxes([[0, 0, 100, 100], [1000, 0, 1100, 100], [2000, 0, 2100, 100]])
    with pytest.raises(GastError, match='capacity'):
        Tk.host_tracks(*Tk.DeviceSort(capacity=2).update_chunk(*R.pack([three])))
    # an infinite predicted box: x[3] = 0 makes h = s / 0
    cap = 8
    trk = Tk.DeviceSort(capacity=cap)
    Tk.host_tracks(*trk.update_chunk(*R.pack([one])))
    x0 = _header_offsets(cap)
    trk.state[x0 + 24:x0 + 32] = torch.zeros(8, dtype=torch.uint8, device='cuda')
    with pytest.raises(GastError, match='infinite'):
        Tk.host_tracks(*trk.update_chunk(*R.pack([one])))
    # the drop-in raises where the reference raises
    from device.lib.track.sort import Sort
    s = Sort()
    frames = R.scenarios()['zero_den'][2]
    s.update(frames[0])
    s.update(frames[1])
    with pytest.raises(GastError, match='IoU'):
        s.update(frames[2])


def test_refusals_before_launch():
    with pytest.raises(GastError):
        Tk.DeviceSort(capacity=0)
    with pytest.raises(GastError):
        Tk.DeviceSort(capacity=5000)
    trk = Tk.DeviceSort(2)
    b, n = R.pack([R._boxes([[0, 0, 100, 100]])])
    with pytest.raises(GastError):
        trk.update_chunk(b, n)                                      # one sequence's boxes for two
    with pytest.raises(GastError):
        trk.update_chunk(np.stack([b, b]).astype(np.float64), np.stack([n, n]))
    with pytest.raises(GastError):
        trk.update_chunk(np.zeros((2, 1, 1, 5), np.float32), np.zeros((2, 1), np.int32))
    with pytest.raises(GastError):
        trk.update_chunk(np.stack([b, b]), n)
    with pytest.raises(GastError, match='shared memory'):
        Tk.DeviceSort(capacity=4096).update_chunk(np.zeros((1, 100, 4), np.float32), np.zeros(1, np.int32))


def test_no_host_synchronisation_and_the_current_stream():
    frames = R.random_sequence(200, 3)
    boxes, counts = R.pack(frames)
    want = Tk.host_tracks(*Tk.DeviceSort().update_chunk(boxes, counts))
    b = torch.from_numpy(boxes).cuda()
    c = torch.from_numpy(counts).cuda()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        trk = Tk.DeviceSort()
        held = (b.clone(), c.clone())
        b.fill_(float('nan'))
        c.zero_()
        torch.cuda._sleep(2_000_000_000)
        b.copy_(held[0])
        c.copy_(held[1])
        torch.cuda.set_sync_debug_mode('error')
        try:
            out = trk.update_chunk(b, c)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert not s.query(), 'update_chunk synchronised with the host'
        got = Tk.host_tracks(*out)
    s.synchronize()
    assert _bits(got) == _bits(want)


def test_zz_report_near_halves():
    print('\nboxes within %g of a round(v, 2) half: %d' % (HALF_TOL, len(NEAR_HALF)))
