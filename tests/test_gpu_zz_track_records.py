"""SORT's tracks to crop records on the device (gast_b200.keypoints2d.track_records / record_inverse,
csrc/records.cuh) against the numpy restatement (tests/recordsref.py) and the host functions, bit for bit; the
device path of video_keypoints against its list path; its refusals, its one synchronisation and stream order."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import keypoints2dref as KR                                         # noqa: E402
import recordsref as R                                              # noqa: E402
import sortref as SR                                                # noqa: E402
from gast_b200 import detection as Dt                               # noqa: E402
from gast_b200 import keypoints2d as K                              # noqa: E402
from gast_b200 import tracking as Tk                                # noqa: E402
from gast_b200.engine import GastError                              # noqa: E402
from test_gpu_zz_keypoints2d import _StandInNet, _clip              # noqa: E402

pytestmark = pytest.mark.gpu
FRAME = (1920, 1080)


def _sort(frames, S=1, chunks=None):
    """DeviceSort over per-frame detections (one list per sequence); the concatenated (rows, counts, status)"""
    trk = Tk.DeviceSort(S, 1, 3, 64)
    packed = [SR.pack(f, 16) for f in frames]
    boxes, counts = np.stack([p[0] for p in packed]), np.stack([p[1] for p in packed])
    if S == 1:
        boxes, counts = boxes[0], counts[0]
    out, t0 = [], 0
    for k in (chunks or [boxes.shape[-3]]):
        out.append(trk.update_chunk(boxes[..., t0:t0 + k, :, :], counts[..., t0:t0 + k], True))
        t0 += k
    return out


def _host(x):
    return x.cpu().numpy()


def _check_records(rec, rows, counts, status, num_person, img=K.IMAGE_SIZE, hm=(72, 96)):
    R4 = rows[None] if rows.dim() == 3 else rows
    N2 = counts[None] if counts.dim() == 1 else counts
    ref = R.track_records(_host(R4), _host(N2), _host(status), num_person, FRAME, img, hm)
    summary = _host(rec.summary)
    assert summary.tolist() == ref['summary'].tolist()
    n = int(_host(rec.total)[0])
    assert n == len(ref['frame']) == summary[:, 0].sum()
    assert _host(rec.frame[:n]).tolist() == ref['frame'].tolist()
    assert _host(rec.slot[:n]).tolist() == ref['slot'].tolist()
    assert _host(rec.forward[:n]).tobytes() == ref['forward'].tobytes()
    assert _host(rec.center[:n]).tobytes() == ref['center'].tobytes()
    assert _host(rec.scale[:n]).tobytes() == ref['scale'].tobytes()
    assert _host(K.record_inverse(rec, hm)[:n]).tobytes() == ref['inverse'].tobytes()
    return ref, n


@pytest.mark.parametrize('num_person', [1, 2, 3])
def test_records_equal_the_restatement_and_the_host_functions(num_person):
    frames = SR.random_sequence(120, seed=num_person, max_persons=6)
    rows, counts, status = _sort([frames])[0]
    rec = K.track_records(rows, counts, status, num_person, FRAME)
    ref, n = _check_records(rec, rows, counts, status, num_person)
    assert n > 100
    word = int(ref['summary'][0, 2])
    if num_person == 3:
        assert word & K.REC_TRACKS and ref['summary'][0, 3] >= 0
        return
    assert word == 0
    if K._cv2 is None:
        return
    lists = Tk.host_tracks(rows, counts, status)
    r = 0
    fwd = _host(rec.forward)
    inv = _host(K.record_inverse(rec, (72, 96)))
    cs = _host(rec.center_scale)
    for t, tr in enumerate(lists):
        sel = K.select_tracks(tr, num_person)
        for box in (sel[:num_person] if sel is not None else ()):
            c, s = K.center_scale(box, FRAME[1], FRAME[0])
            f, i = K.affine_pair(c, s, K.IMAGE_SIZE, (72, 96))
            assert cs[r].tobytes() == np.concatenate([c, s]).tobytes()
            assert fwd[r].tobytes() == f.tobytes() and inv[r].tobytes() == i.tobytes(), (t, r)
            r += 1
    assert r == n


def test_sequences_in_one_launch_and_split_chunks():
    seqs = [SR.random_sequence(90, seed=20 + s, max_persons=5) for s in range(4)]
    rows, counts, status = _sort(seqs, S=4)[0]
    rec = K.track_records(rows, counts, status, 2, FRAME)
    ref, n = _check_records(rec, rows, counts, status, 2)
    at = 0
    for s in range(4):
        one = K.track_records(*_sort([seqs[s]])[0], 2, FRAME)
        m = int(_host(one.total)[0])
        assert _host(one.summary)[0].tolist() == _host(rec.summary)[s].tolist()
        assert torch.equal(one.frame[:m] + s * 90, rec.frame[at:at + m])
        for a, b in ((one.slot, rec.slot), (one.forward, rec.forward), (one.center_scale, rec.center_scale)):
            assert torch.equal(a[:m], b[at:at + m])
        at += m
    assert at == n
    # K in uneven chunks: the same records, frames and slots offset by the chunks before
    whole = K.track_records(*_sort([seqs[1]])[0], 2, FRAME)
    m = int(_host(whole.total)[0])
    parts, t0, kept = [], 0, 0
    for (r, c, st), k in zip(_sort([seqs[1]], chunks=[17, 5, 1, 67]), [17, 5, 1, 67]):
        p = K.track_records(r, c, st, 2, FRAME)
        q = int(_host(p.total)[0])
        parts.append((p.frame[:q] + t0, p.slot[:q] + 2 * kept, p.forward[:q], p.center_scale[:q]))
        t0 += k
        kept += int(_host(p.summary)[0, 1])
    for j, w in enumerate((whole.frame, whole.slot, whole.forward, whole.center_scale)):
        assert torch.equal(torch.cat([p[j] for p in parts]), w[:m])
    again = K.track_records(*_sort([seqs[1]])[0], 2, FRAME)                  # a repeat gives the same bits
    assert torch.equal(again.summary, whole.summary) and torch.equal(again.forward[:m], whole.forward[:m])


def _triple(boxes, cap=4):
    """a per-frame track list (None: skipped) as update_chunk's (rows, counts, status) on the device"""
    T = len(boxes)
    rows = np.zeros((T, cap, 5))
    counts = np.full(T, -1, np.int32)
    for t, b in enumerate(boxes):
        if b is not None:
            counts[t] = len(b)
            rows[t, :len(b)] = b
    dev = torch.device('cuda')
    return (torch.from_numpy(rows).to(dev), torch.from_numpy(counts).to(dev),
            torch.zeros(1, dtype=torch.int32, device=dev))


def _same_call(frames, triple, num_person):
    net_d, net_h = _StandInNet().cuda(), _StandInNet().cuda()
    kd, sd = K.video_keypoints(frames, triple, net_d, num_person)
    kh, sh = K.video_keypoints(frames, Tk.host_tracks(*triple), net_h, num_person)
    assert torch.equal(kd, kh) and torch.equal(sd, sh)
    assert len(net_d.seen) == len(net_h.seen)
    for (xd, yd), (xh, yh) in zip(net_d.seen, net_h.seen):
        assert torch.equal(xd, xh) and torch.equal(yd, yh)
    return kd


@pytest.mark.parametrize('num_person', [1, 2])
def test_video_keypoints_device_path_equals_the_list_path(num_person):
    frames, boxes = _clip()
    kd = _same_call(torch.from_numpy(frames).cuda(), _triple(boxes), num_person)
    assert kd.shape[1] == 4
    _same_call(frames, _triple(boxes), num_person)               # numpy frames
    seq = SR.random_sequence(40, seed=7, max_persons=4)
    frames = KR.synth_frames(40, FRAME[1], FRAME[0], seed=3)
    _same_call(torch.from_numpy(frames).cuda(), _sort([seq])[0], num_person)


class _Detector:
    """a stand-in for Darknet: two persons walking across each letterboxed frame, fixed predictions per frame"""

    def __init__(self, T, D=416):
        n = Dt.num_predictions(D)
        p = np.zeros((T, n, 85), np.float32)
        for t in range(T):
            for i in range(2):
                p[t, i, :5] = [80 + 3 * t + 170 * i, 200 + i * 7, 60 + i, 150, 0.9]
                p[t, i, 5] = 0.95
        self.p = torch.from_numpy(p).cuda()

    def __call__(self, x, cuda):
        return self.p[:x.shape[0]]


def test_video_boxes_on_device_chain_equals_the_host_chain():
    T = 24
    frames = torch.from_numpy(KR.synth_frames(T, 540, 960, seed=5)).cuda()
    det = _Detector(T)
    triple = Dt.video_boxes(frames, det, Tk.DeviceSort(), on_device=True)
    assert isinstance(triple, tuple) and all(x.is_cuda for x in triple)
    lists = Dt.video_boxes(frames, det, Tk.DeviceSort())
    for a, b in zip(Tk.host_tracks(*triple), lists):
        assert (a is None and b is None) or a.tobytes() == b.tobytes()
    for num_person in (1, 2):
        net_d, net_h = _StandInNet().cuda(), _StandInNet().cuda()
        kd, sd = K.video_keypoints(frames, triple, net_d, num_person)
        kh, sh = K.video_keypoints(frames, lists, net_h, num_person)
        assert kd.shape[1] == T and torch.equal(kd, kh) and torch.equal(sd, sh)
        assert torch.equal(net_d.seen[0][0], net_h.seen[0][0])
    with pytest.raises(GastError, match='DeviceSort'):
        Dt.video_boxes(frames, det, SR.Sort(), on_device=True)


def _message(call):
    with pytest.raises(GastError) as e:
        call()
    return str(e.value)


def test_refusals_carry_the_host_paths_messages():
    frames, boxes = _clip()
    frames = torch.from_numpy(frames).cuda()
    net = _StandInNet().cuda()
    cases = []
    b = [None if x is None else x.copy() for x in boxes]
    b[2][0, 1] = np.nan                                            # a NaN box
    cases.append((b, 2))
    b = [None if x is None else x.copy() for x in boxes]
    b[5][1, 2:4] = b[5][1, :2] - 3                                 # a box with no width and no height
    cases.append((b, 2))
    cases.append((boxes, 3))                                       # two tracks in frame 0 for three persons
    for b, num_person in cases:
        triple = _triple(b)
        want = _message(lambda: K.video_keypoints(frames, Tk.host_tracks(*triple), net, num_person))
        assert 'keypoints2d' in want
        assert _message(lambda: K.video_keypoints(frames, triple, net, num_person)) == want
    for word in (1, 2, 4, 8, 16, 4 | 8):                           # SORT's status words
        rows, counts, status = _triple(boxes)
        status.fill_(word)
        want = _message(lambda: Tk.host_tracks(rows, counts, status))
        assert _message(lambda: K.video_keypoints(frames, (rows, counts, status), net, 2)) == want


def test_synchronisation():
    frames, boxes = _clip()
    frames = torch.from_numpy(frames).cuda()
    triple = _triple(boxes)
    net = _StandInNet().cuda()
    K.video_keypoints(frames, triple, net, 2)                      # warm up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        rec = K.track_records(*triple, 2, (960, 540))
        inv = K.record_inverse(rec, (72, 96))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert inv.shape == (6 * 2, 2, 3)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            kp, sc = K.video_keypoints(frames, triple, net, 2)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in caught if 'synchroniz' in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in caught]
    assert kp.shape == (2, 4, 17, 2)


# stream order: the pattern of test_gpu_zz_cuda_streams.py part A, for the two new entries
def _sleep(ms):
    n = 20_000_000
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(n)
    e1.record()
    e1.synchronize()
    torch.cuda._sleep(int(n / e0.elapsed_time(e1) * ms))


def _ordered(make, run):
    """run(make()) on the default stream, then on a side stream with make()'s tensors NaN (integers 0) until a
    device sleep ends; the call must return while the stream sleeps and give the same bits"""
    held = make()
    want = [_host(x) for x in run(held)]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        held = make()
        saved = [t.clone() for t in held]
        for t in held:
            t.fill_(float('nan') if t.is_floating_point() else 0)
        _sleep(200)
        for t, v in zip(held, saved):
            t.copy_(v)
        out = run(held)
        assert not s.query(), 'synchronised with the host'
    s.synchronize()
    got = [_host(x) for x in out]
    assert len(got) == len(want) and all(a.tobytes() == b.tobytes() for a, b in zip(got, want))


def test_stream_order():
    rows, counts, status = _sort([SR.random_sequence(60, seed=3, max_persons=5)])[0]
    rec = K.track_records(rows, counts, status, 2, FRAME)
    n = int(_host(rec.total)[0])
    assert n > 50

    def records(h):
        r = K.track_records(*h, 2, FRAME)
        return [r.summary, r.total, r.frame[:n], r.slot[:n], r.forward[:n], r.center_scale[:n]]
    _ordered(lambda: [rows.clone(), counts.clone(), status.clone()], records)
    cs, total = rec.center_scale.clone(), rec.total.clone()
    _ordered(lambda: [cs.clone(), total.clone()],
             lambda h: [K.record_inverse(K.TrackRecords(None, None, None, h[0], None, h[1]), (72, 96))[:n]])
