"""The live tick (gast_b200.live.LiveTick, csrc/live.cuh) against the eager composition of the existing calls, bit
for bit: letterbox -> Darknet -> person_boxes -> DeviceSort.update_chunk -> host_tracks -> the host geometry without
rounding -> crop_persons -> HRNet -> decode_heatmaps -> device.tools.preprocess -> PoseStream.push of the streams the
restated slot rule (tests/liveref.py) picks -> camera_to_world -> revise_skes_real_time of the active persons.  Also
the graphed tick against the eager one, repeat runs, no host synchronisation, stream order, the status word, the
refusals and the weight-change rule."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import detectionref as DR                                           # noqa: E402
import liveref as LR                                                # noqa: E402
import sortref as SR                                                # noqa: E402
from common.graph_utils import adj_mx_from_skeleton                 # noqa: E402
from common.skeleton import Skeleton                                # noqa: E402
from device.tools import preprocess as DP                           # noqa: E402
from gast_b200 import _lib as L                                     # noqa: E402
from gast_b200 import detection as Dt                               # noqa: E402
from gast_b200 import keypoints2d as K                              # noqa: E402
from gast_b200 import pipeline as Pp                                # noqa: E402
from gast_b200 import synth                                         # noqa: E402
from gast_b200 import tracking as Tk                                # noqa: E402
from gast_b200.engine import GastError                              # noqa: E402
from gast_b200.live import LiveTick                                 # noqa: E402
from gast_b200.realtime import PoseStream                           # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f          # noqa: E402
from test_gpu_zz_keypoints2d import _StandInNet                     # noqa: E402

pytestmark = pytest.mark.gpu
W, H, D = 640, 360, 416


def _model(causal=True, seed=3):
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    m = SpatioTemporalModelOptimized1f(adj, 17, 2, 17, [3, 3, 3], causal=causal, channels=32)
    synth.randomize_module(m, seed)
    return m.cuda().eval()


class _Darknet:
    """a stand-in for Darknet that returns the predictions the test set for this tick (`preds` (C, N, 85)); the
    letterboxed input enters through a zero term"""

    def __init__(self, C):
        self.preds = torch.zeros((C, DR.num_predictions(D), 85), dtype=torch.float32, device='cuda')

    def __call__(self, x, cuda):
        return self.preds + x[:, :1, :1, :1].reshape(-1, 1, 1) * 0


class _Pose(_StandInNet):
    """the keypoint test's stand-in HRNet, without its record of inputs"""

    def forward(self, x):
        y = super().forward(x)
        self.seen.clear()
        return y


def _predictions(frames_boxes, seed):
    """(C, N, 85) float32: each camera's boxes (hundredths of 1920 x 1080 pixels) as detections of a 640 x 360 frame"""
    out = []
    sf = D / W
    py = (D - H * sf) / 2
    for c, rows in enumerate(frames_boxes):
        p = DR.background(D, seed * 7 + c)
        for i, b in enumerate(np.asarray(rows, np.float64).reshape(-1, 4)):
            x1, y1, x2, y2 = b / 100 / 3
            DR.put(p, 50 + 97 * i, (x1 + x2) / 2 * sf, (y1 + y2) / 2 * sf + py, (x2 - x1) * sf, (y2 - y1) * sf,
                   0.99 - 0.01 * i)
        out.append(p)
    return torch.from_numpy(np.stack(out)).cuda()


def _scene(C, T, seed):
    """T ticks of C cameras: walking persons, some ticks empty, some crowded"""
    seqs = [SR.random_sequence(T, seed=seed * 10 + c, max_persons=8) for c in range(C)]
    ticks = []
    for t in range(T):
        rows = [np.zeros((0, 4)) if (t + c) % 23 == 5 else seqs[c][t] for c in range(C)]
        ticks.append(_predictions(rows, seed * 1000 + t))
    frames = torch.from_numpy(DR.synth_frames(C, H, W, seed=seed)).cuda()
    return frames, ticks


class _Glue:
    """the eager composition of the existing calls, one tick at a time"""

    def __init__(self, det, pose, model, C, P, augment):
        self.det, self.pose, self.C, self.P = det, pose, C, P
        self.sort = Tk.DeviceSort(C, 1, 3, 256)
        self.ps = PoseStream(model, C * P, augment=augment)
        self.books = [LR.SlotBook(P) for _ in range(C)]
        self.tick = 0

    def __call__(self, frames):
        C, P, n = self.C, self.P, self.C * self.P
        pred = self.det(Dt.letterbox(frames, D), True)
        boxes, _, counts = Dt.person_boxes(pred, (W, H), D, 0.7, 0.4, Dt.MAX_DET)
        rows, cnt, st = self.sort.update_chunk(boxes[:, None], counts[:, None], True)
        tracks = Tk.host_tracks(rows, cnt, st)
        box = np.zeros((n, 4))
        sel = np.zeros(n, bool)
        for c in range(C):
            tr = tracks[c][0]
            k = -1 if tr is None else len(tr)
            pick, _ = LR.select(k, P, 256)
            slots = self.books[c].assign([int(tr[r, 4]) for r in pick], self.tick)
            for r, s in zip(pick, slots):
                box[c * P + s] = tr[r, :4]
                sel[c * P + s] = True
        _, _, fwd, inv, bits = LR.slot_geometry(box, H, W, K.IMAGE_SIZE, (72, 96))
        slot_ok = sel & (bits == 0)
        crops = K.crop_persons(frames, np.arange(n) // P, fwd, K.IMAGE_SIZE)
        kp, mv = K.decode_heatmaps(self.pose(crops), inv)
        hk, hs, frames_v = DP.h36m_coco_format(kp[:, None], mv.view(n, 1, 17))
        kept = [s for s in range(n) if (kp[s] != 0).any()]
        kpts = torch.zeros((n, 17, 2), device='cuda')
        scores = torch.zeros((n, 17), device='cuda')
        active = np.zeros(n, bool)
        if kept:
            re = DP.revise_kpts(hk, hs, frames_v)
            for q, s in enumerate(kept):
                if slot_ok[s] and frames_v[q].numel() == 1:
                    active[s] = True
                    kpts[s], scores[s] = re[q, 0], hs[q, 0]
        poses = torch.zeros((n, 17, 3), device='cuda')
        streams = np.flatnonzero(active)
        fresh = [s for s in streams if self.books[s // P].fresh[s % P]]
        if fresh:
            self.ps.reset(fresh)
        for s in streams:
            self.books[s // P].fresh[s % P] = False
        if streams.size:
            x = Pp.normalize_screen(kpts[torch.from_numpy(streams).cuda()], W, H)
            y, _ = self.ps.push(x, streams=streams)
            world = Pp.camera_to_world(y, LR.ROT, 0)
            for c in range(C):
                mine = [q for q, s in enumerate(streams) if s // P == c]
                if mine:
                    idx = torch.tensor(mine).cuda()
                    placed = DP.revise_skes_real_time(world[idx], kpts[torch.from_numpy(streams[mine]).cuda()], W)
                    poses[torch.from_numpy(streams[mine]).cuda()] = placed
        self.tick += 1
        ids = np.concatenate([b.ids for b in self.books])
        return dict(poses=poses, keypoints=kpts, scores=scores, ids=ids, active=active)


def _same(out, ref, C, P):
    assert out.poses.cpu().numpy().tobytes() == ref['poses'].view(C, P, 17, 3).cpu().numpy().tobytes()
    assert out.keypoints.cpu().numpy().tobytes() == ref['keypoints'].view(C, P, 17, 2).cpu().numpy().tobytes()
    assert out.scores.cpu().numpy().tobytes() == ref['scores'].view(C, P, 17).cpu().numpy().tobytes()
    assert out.ids.cpu().numpy().reshape(-1).tolist() == ref['ids'].tolist()
    assert out.active.cpu().numpy().reshape(-1).tolist() == ref['active'].tolist()


def _snapshot(out):
    return [t.clone() for t in (out.poses, out.keypoints, out.scores, out.ids, out.active)]


@pytest.mark.parametrize('C,P,augment', [(1, 1, False), (1, 2, True), (3, 1, True), (3, 2, False), (3, 2, True),
                                         (1, 1, True), (1, 2, False), (3, 1, False)])
def test_tick_equals_the_composition_and_the_graph_equals_eager(C, P, augment):
    T = 200
    frames, ticks = _scene(C, T, seed=C * 10 + P)
    model = _model()
    det, pose = _Darknet(C), _Pose().cuda()
    eager = LiveTick(det, pose, model, C, (W, H), num_person=P, augment=augment)
    graphed = LiveTick(det, pose, model, C, (W, H), num_person=P, augment=augment, graph=True)
    glue = _Glue(det, pose, model, C, P, augment)
    active = 0
    for t in range(T):
        det.preds.copy_(ticks[t])
        a = _snapshot(eager(frames))
        b = graphed(frames)
        assert all(torch.equal(x, y) for x, y in zip(a, _snapshot(b)))
        ref = glue(frames)
        _same(b, ref, C, P)
        active += int(ref['active'].sum())
    assert graphed.graph is not None and active > T * C * P // 4
    assert (eager.status()[0] == 0).all()


def test_two_runs_repeat_and_no_tick_synchronises():
    C, P, T = 3, 2, 40
    frames, ticks = _scene(C, T, seed=7)
    model = _model()
    runs = []
    for graph in (False, True, False):
        det, pose = _Darknet(C), _Pose().cuda()
        tick = LiveTick(det, pose, model, C, (W, H), num_person=P, augment=True, graph=graph)
        outs = []
        for t in range(T):
            det.preds.copy_(ticks[t])
            if t >= 2:
                torch.cuda.synchronize()
                torch.cuda.set_sync_debug_mode('error')
            try:
                out = tick(frames)
            finally:
                torch.cuda.set_sync_debug_mode(0)
            outs.append([x.cpu() for x in _snapshot(out)])
        runs.append(outs)
        assert tick.last_launches >= 11
    for r in runs[1:]:
        assert all(torch.equal(x, y) for a, b in zip(runs[0], r) for x, y in zip(a, b))


def _sleep(ms):
    n = 20_000_000
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    torch.cuda._sleep(n)
    e1.record()
    e1.synchronize()
    torch.cuda._sleep(int(n / e0.elapsed_time(e1) * ms))


@pytest.mark.parametrize('graph', [False, True])
def test_stream_order(graph):
    C, P = 2, 2
    frames, ticks = _scene(C, 4, seed=11)
    model = _model()
    want = []
    for side in (False, True):
        det, pose = _Darknet(C), _Pose().cuda()
        tick = LiveTick(det, pose, model, C, (W, H), num_person=P, graph=graph)
        for t in range(3):
            det.preds.copy_(ticks[t])
            tick(frames)
        torch.cuda.synchronize()
        if not side:
            det.preds.copy_(ticks[3])
            want = [x.cpu() for x in _snapshot(tick(frames))]
            continue
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            held = frames.clone()
            frames.zero_()
            det.preds.fill_(float('nan'))
            _sleep(200)
            frames.copy_(held)
            det.preds.copy_(ticks[3])
            out = tick(frames)
            assert not s.query(), 'synchronised with the host'
        s.synchronize()
        got = [x.cpu() for x in _snapshot(out)]
        assert all(torch.equal(x, y) for x, y in zip(got, want))


def _slots(rows, counts, sort_status, P, book, status, hm=(72, 96)):
    n = counts.numel() * P
    dev = 'cuda'
    act = torch.zeros(n, dtype=torch.int32, device=dev)
    fwd = torch.zeros((n, 6), dtype=torch.float64, device=dev)
    inv = torch.zeros((n, 6), dtype=torch.float64, device=dev)
    cs = torch.zeros((n, 4), dtype=torch.float32, device=dev)
    p = lambda t: C.c_void_p(t.data_ptr())                           # noqa: E731
    rc = L.load().gast_live_slots(p(rows), p(counts), p(sort_status), counts.numel(), rows.shape[1], P, W, H, 288, 384,
                                  hm[0], hm[1], p(book), p(status), p(act), p(fwd), p(inv), p(cs),
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, L.last_error()
    return act, fwd, inv, cs


def test_every_status_cause_sets_its_bit_and_first_tick():
    P, cap = 3, 4
    book = torch.tensor([-1, -1, 1], dtype=torch.int64, device='cuda')[:, None].repeat(1, 4 * P).contiguous()
    status = torch.full((4, 16), -1, dtype=torch.int64, device='cuda')
    status[:, :2] = 0
    ok = [[10.0, 20.0, 110.0, 220.0, 1.0], [30.0, 40.0, 130.0, 240.0, 2.0], [50.0, 60.0, 150.0, 260.0, 3.0],
          [0.0, 0.0, 0.0, 0.0, 0.0]]
    rows = torch.tensor([ok] * 4, dtype=torch.float64, device='cuda')
    counts = torch.tensor([3, 3, 3, 3], dtype=torch.int32, device='cuda')
    sort_status = torch.zeros(4, dtype=torch.int32, device='cuda')
    act, *_ = _slots(rows, counts, sort_status, P, book, status)
    assert act.tolist() == [1] * 12 and status[:, 0].tolist() == [0] * 4 and status[:, 1].tolist() == [1] * 4
    rows[1, 1, 0] = float('nan')                 # a non-finite box
    rows[2, 0, 2], rows[2, 0, 3] = 10.0, 20.0    # an empty box
    counts[0] = 2                                # 2 <= k < num_person
    sort_status[3] = 4                           # SORT's IoU bit
    act, *_ = _slots(rows, counts, sort_status, P, book, status)
    st = status.cpu().numpy()
    # a non-finite box gives a non-finite matrix too, as in gast_track_records
    assert st[:, 0].tolist() == [K.REC_TRACKS, K.REC_NONFINITE | K.REC_MATRIX, K.REC_EMPTY, 4]
    assert st[0, 2 + 8] == 1 and st[1, 2 + 9] == st[1, 2 + 11] == 1 and st[2, 2 + 10] == 1 and st[3, 2 + 2] == 1
    assert act.view(4, P).tolist() == [[0, 0, 0], [1, 0, 1], [1, 1, 0], [1, 1, 1]]
    _slots(rows, counts, sort_status, P, book, status)
    st2 = status.cpu().numpy()
    assert (st2[:, 2:] == st[:, 2:]).all() and st2[:, 1].tolist() == [3] * 4     # sticky, first tick kept


def test_check_raises_the_host_messages_and_reset_clears():
    model = _model()
    tick = LiveTick(_Darknet(2), _Pose().cuda(), model, 2, (W, H), num_person=2)
    tick.check()
    tick._status[1, 0] = 2
    with pytest.raises(GastError, match='tracking: sequence 1: the tracker list outgrew its capacity'):
        tick.check()
    tick._status[1, 0] = K.REC_NONFINITE
    tick._status[1, 2 + 9] = 5
    with pytest.raises(GastError, match='camera 1 tick 5: a box that is not finite'):
        tick.check()
    tick.reset([1])
    tick.check()
    assert tick.out.ids.tolist() == [[-1, -1], [-1, -1]]


def test_refusals_come_before_any_launch_and_weights_follow_the_rule():
    C, P = 2, 2
    frames, ticks = _scene(C, 3, seed=5)
    det, pose = _Darknet(C), _Pose().cuda()
    with pytest.raises(GastError, match='causal'):
        LiveTick(det, pose, _model(causal=False), C, (W, H))
    m = _model()
    m.train()
    with pytest.raises(GastError, match='eval'):
        LiveTick(det, pose, m, C, (W, H))
    m.eval()
    for graph in (False, True):
        tick = LiveTick(det, pose, m, C, (W, H), num_person=P, graph=graph)
        det.preds.copy_(ticks[0])
        tick(frames)
        torch.cuda.synchronize()
        before = tick._status.clone()
        for bad in (frames[:1], frames.float(), frames[:, :, :-1].contiguous(), frames.cpu()):
            with pytest.raises(GastError, match='frames'):
                tick(bad)
        for call in (lambda: tick.export_streams([0]), lambda: tick.import_streams(None, [0]),
                     lambda: tick.push(None), lambda: tick.peek()):
            with pytest.raises(GastError):
                call()
        m.train()
        with pytest.raises(GastError, match='eval'):
            tick(frames)
        m.eval()
        with torch.no_grad():
            next(m.parameters()).mul_(1.0001)
        with pytest.raises(GastError, match='reset'):
            tick(frames)
        assert torch.equal(tick._status, before)
        tick.reset()
        det.preds.copy_(ticks[1])
        tick(frames)
        assert int(tick._status[0, 1]) == 2


def test_a_net_that_cannot_be_captured_is_refused_at_construction():
    pose = _Pose().cuda()

    class _Uncapturable(torch.nn.Module):
        def forward(self, x):
            return pose(x) + float(x.sum().item()) * 0

    with pytest.raises(GastError, match='cannot be captured'):
        LiveTick(_Darknet(1), _Uncapturable(), _model(), 1, (W, H), graph=True)
    LiveTick(_Darknet(1), _Uncapturable(), _model(), 1, (W, H))                # eager ticks take it
