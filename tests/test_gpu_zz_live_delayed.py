"""The delayed live tick of the non-causal models (gast_b200.live.LiveTick with a non-causal model, csrc/live.cuh's
gast_live_delayed_*) against the eager composition of the existing calls, bit for bit: test_gpu_zz_live's glue up to
the stream inputs, then PoseStream.peek(latency, streams=ending) -> reset(ending) -> PoseStream.push(streams=active) ->
PoseStream.peek(latency - L, streams=active) -> camera_to_world -> revise_skes_real_time of each group with the
keypoints of each pose's own frame (kept on the host, tests/livedelayedref.py's bookkeeping).  Also the graphed tick
against the eager one, tails against end() plus held pushes, end(cameras), the link to the reference's gen_pose
(tta.evaluate_sequence of one person's sequence), repeat runs, no host synchronisation, stream order, the refusals
and the weight-change rule."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import detectionref as DR                                           # noqa: E402
import livedelayedref as LD                                         # noqa: E402
import liveref as LR                                                # noqa: E402
from common.graph_utils import adj_mx_from_skeleton                 # noqa: E402
from common.skeleton import Skeleton                                # noqa: E402
from device.tools import preprocess as DP                           # noqa: E402
from gast_b200 import engine                                        # noqa: E402
from gast_b200 import pipeline as Pp                                # noqa: E402
from gast_b200 import synth, tta                                    # noqa: E402
from gast_b200.engine import GastError                              # noqa: E402
from gast_b200.live import LiveTick                                 # noqa: E402
from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f   # noqa: E402
from test_gpu_zz_delayed_stream import WHOLE_BAR                    # noqa: E402
from test_gpu_zz_live import (D, H, W, _Darknet, _Glue, _Pose, _predictions, _scene,    # noqa: E402,F401
                              _sleep)

pytestmark = pytest.mark.gpu


def _model(kind='opt', fw=(3, 3, 3), seed=3, channels=32):
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    if kind == 'dilated':
        m = SpatioTemporalModel(adj, 17, 2, 17, list(fw), channels=channels)
    else:
        m = SpatioTemporalModelOptimized1f(adj, 17, 2, 17, list(fw), causal=False, channels=channels)
    synth.randomize_module(m, seed)
    return m.cuda().eval()


class _Recorder(object):
    """stands in for _Glue's PoseStream: records the restarting streams, the pushed streams and their input rows"""

    def reset(self, streams):
        self.fresh = list(streams)

    def push(self, x, streams):
        self.x, self.streams = x, np.asarray(streams)
        return torch.zeros((len(streams), 17, 3), device='cuda'), None


class _DelayedGlue(_Glue):
    """test_gpu_zz_live's glue up to the stream inputs, then the delayed composition.  flush='peek': a tail is
    PoseStream.peek(latency) before reset; flush='end': PoseStream.end plus latency held pushes of the same streams"""

    def __init__(self, det, pose, model, C, P, augment, lookahead=None, max_gap=None, flush='peek'):
        super().__init__(det, pose, model, C, P, augment)
        self.real = self.ps
        self.lat, self.L, self.flush = self.real.latency, lookahead, flush
        self.seqs = LD.Sequences(C * P, self.lat, lookahead, max_gap)
        self.hist = [[] for _ in range(C * P)]        # (keypoints, tick) of each slot's current sequence's frames

    def _placed(self, y, slots, pos, hist, one_by_one=False):
        """camera_to_world of y (m, 17, 3) and revise_skes_real_time with each pose's own frame's keypoints, per camera
        over the group or pose by pose -> (poses (m, 17, 3), ticks (m,))"""
        world = Pp.camera_to_world(y, LR.ROT, 0)
        kp = torch.stack([hist[s][p][0] for s, p in zip(slots, pos)])
        ticks = np.array([hist[s][p][1] for s, p in zip(slots, pos)], np.int64)
        out = torch.zeros_like(world)
        groups = [[i] for i in range(len(slots))] if one_by_one else \
            [[i for i, s in enumerate(slots) if s // self.P == c] for c in range(self.C)]
        for g in groups:
            if g:
                idx = torch.tensor(g).cuda()
                out[idx] = DP.revise_skes_real_time(world[idx], kp[idx], W)
        return out, ticks

    def _tails(self, ending, pos):
        """the placed tails of the ending slots, with their rows' positions pos (n, latency)"""
        n, lat = self.C * self.P, self.lat
        tail = torch.zeros((n, lat, 17, 3), device='cuda')
        frame = np.full((n, lat), -1, np.int64)
        s = np.flatnonzero(ending)
        if s.size:
            if self.flush == 'peek':
                y, index = self.real.peek(lat, streams=s)
            else:
                self.real.end(s)
                y, index = self.real.push_frames(torch.full((s.size, lat, 17, 2), float('nan'), device='cuda'),
                                                 streams=s)
            assert np.array_equal(index.numpy(), pos[s])
            rows = [(q, k) for q in range(s.size) for k in range(lat) if pos[s[q], k] >= 0]
            if rows:
                yy = torch.stack([y[q, k] for q, k in rows])
                placed, ticks = self._placed(yy, [s[q] for q, _ in rows], [pos[s[q], k] for q, k in rows], self.hist,
                                             one_by_one=True)
                for i, (q, k) in enumerate(rows):
                    tail[s[q], k] = placed[i]
                    frame[s[q], k] = ticks[i]
        return tail, frame

    def __call__(self, frames):
        C, P, n, lat = self.C, self.P, self.C * self.P, self.lat
        t = self.tick
        rec = self.ps = _Recorder()
        rec.fresh, rec.streams = [], np.zeros(0, np.int64)
        ref = super().__call__(frames)
        self.ps = self.real
        active = ref['active']
        restart = np.zeros(n, bool)
        restart[rec.fresh] = True
        out = self.seqs.tick(t, active, ref['ids'], restart)
        ending = out['ending']
        tail, tail_frame = self._tails(ending, out['tail'])
        start = ending | out['fresh']
        if start.any():
            self.real.reset(np.flatnonzero(start))
        for s in np.flatnonzero(start):
            self.hist[s] = []
        streams = rec.streams
        assert np.array_equal(streams, np.flatnonzero(active))
        kpts = ref['keypoints']
        for s in streams:
            self.hist[s].append((kpts[s].clone(), t))
        poses = torch.zeros((n, 17, 3), device='cuda')
        frame = np.full(n, -1, np.int64)
        now = torch.zeros((n, 17, 3), device='cuda')
        now_frame = np.full(n, -1, np.int64)
        if streams.size:
            y, index = self.real.push(rec.x, streams=streams)
            assert np.array_equal(index.numpy(), out['final'][streams])
            g = [q for q, s in enumerate(streams) if out['final'][s] >= 0]
            if g:
                placed, ticks = self._placed(y[g], streams[g], out['final'][streams[g]], self.hist)
                poses[torch.from_numpy(streams[g]).cuda()] = placed
                frame[streams[g]] = ticks
            if self.L is not None:
                yp, pidx = self.real.peek(lat - self.L, streams=streams)
                assert np.array_equal(pidx.numpy()[:, -1], out['now'][streams])
                g = [q for q, s in enumerate(streams) if out['now'][s] >= 0]
                if g:
                    placed, ticks = self._placed(yp[g, -1], streams[g], out['now'][streams[g]], self.hist)
                    now[torch.from_numpy(streams[g]).cuda()] = placed
                    now_frame[streams[g]] = ticks
        ref.update(poses=poses, frame=frame, tail=tail, tail_frame=tail_frame, tail_ids=out['tail_ids'])
        if self.L is not None:
            ref.update(now=now, now_frame=now_frame)
        return ref

    def end(self, cameras):
        """the composition's flush of the listed cameras' pending sequences -> (tail, tail_frame, tail_ids)"""
        ending, pos, ids = self.seqs.end(cameras, self.P)
        tail, frame = self._tails(ending, pos)
        return tail, frame, ids


FIELDS = ('poses', 'keypoints', 'scores', 'ids', 'active', 'frame', 'now', 'now_frame', 'tail', 'tail_frame',
          'tail_ids')


def _snapshot(out):
    return [None if getattr(out, f) is None else getattr(out, f).clone() for f in FIELDS]


def _same(out, ref, C, P):
    n = C * P
    eq = lambda a, b: a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()   # noqa: E731
    assert eq(out.poses, ref['poses'].view(C, P, 17, 3))
    assert eq(out.keypoints, ref['keypoints'].view(C, P, 17, 2))
    assert eq(out.scores, ref['scores'].view(C, P, 17))
    assert out.ids.cpu().numpy().reshape(-1).tolist() == ref['ids'].tolist()
    assert out.active.cpu().numpy().reshape(-1).tolist() == ref['active'].tolist()
    assert out.frame.cpu().numpy().reshape(-1).tolist() == ref['frame'].tolist()
    assert eq(out.tail, ref['tail'].view(C, P, -1, 17, 3))
    assert out.tail_frame.cpu().numpy().reshape(n, -1).tolist() == ref['tail_frame'].tolist()
    assert out.tail_ids.cpu().numpy().reshape(-1).tolist() == ref['tail_ids'].tolist()
    if 'now' in ref:
        assert eq(out.now, ref['now'].view(C, P, 17, 3))
        assert out.now_frame.cpu().numpy().reshape(-1).tolist() == ref['now_frame'].tolist()
    else:
        assert out.now is None and out.now_frame is None


CASES = [  # C, P, augment, lookahead ('last': latency - 1), model, max_gap, precision
    (1, 1, False, None, ('dilated', (3, 3, 3)), None, 'fp32'),
    (1, 2, True, 0, ('dilated', (3, 3, 3)), 2, 'fp32'),
    (3, 1, True, 'last', ('opt', (3, 3, 3)), None, 'fp32'),
    (3, 2, False, 0, ('opt', (3, 3, 3, 3)), None, 'fp32'),
    (3, 2, True, None, ('opt', (3, 3, 3)), 0, 'fp32'),
    (1, 2, False, 'last', ('opt', (3, 3, 3)), None, 'fp16'),
]


@pytest.mark.parametrize('C,P,augment,L,kind,max_gap,precision', CASES)
def test_tick_equals_the_composition_and_the_graph_equals_eager(C, P, augment, L, kind, max_gap, precision):
    T = 200
    frames, ticks = _scene(C, T, seed=C * 10 + P + 3)
    model = _model(*kind)
    engine.set_precision(model, precision)
    try:
        lat = (model.receptive_field() - 1) // 2
        L = lat - 1 if L == 'last' else L
        det, pose = _Darknet(C), _Pose().cuda()
        kw = dict(num_person=P, augment=augment, lookahead=L, max_gap=max_gap, delayed=True)
        eager = LiveTick(det, pose, model, C, (W, H), **kw)
        graphed = LiveTick(det, pose, model, C, (W, H), graph=True, **kw)
        assert eager.latency == lat
        glue = _DelayedGlue(det, pose, model, C, P, augment, L, max_gap)
        finals = tails = 0
        for t in range(T):
            det.preds.copy_(ticks[t])
            a = _snapshot(eager(frames))
            b = graphed(frames)
            assert all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, _snapshot(b)))
            ref = glue(frames)
            _same(b, ref, C, P)
            finals += int((ref['frame'] >= 0).sum())
            tails += int((ref['tail_frame'] >= 0).sum())
        assert graphed.graph is not None and finals > 0 and tails > 0
        got = graphed.end()
        want = glue.end(list(range(C)))
        assert torch.equal(got[0], want[0].view(C, P, lat, 17, 3))
        assert got[1].cpu().numpy().reshape(C * P, lat).tolist() == want[1].tolist()
        assert got[2].cpu().numpy().reshape(-1).tolist() == want[2].tolist()
    finally:
        engine.set_precision(model, 'fp32')


def test_tails_equal_end_and_held_pushes_and_end_cameras_equals_a_flush():
    C, P, T = 3, 2, 120
    frames, ticks = _scene(C, T, seed=17)
    model = _model()
    lat = (model.receptive_field() - 1) // 2
    det, pose = _Darknet(C), _Pose().cuda()
    tick = LiveTick(det, pose, model, C, (W, H), num_person=P, augment=True, max_gap=1, graph=True,
                    delayed=True)
    glue = _DelayedGlue(det, pose, model, C, P, True, None, 1, flush='end')
    tails = 0
    for t in range(T):
        det.preds.copy_(ticks[t])
        out = tick(frames)
        ref = glue(frames)
        _same(out, ref, C, P)
        tails += int((ref['tail_frame'] >= 0).sum())
    assert tails > lat
    got = [x.clone() for x in tick.end([1])]
    want = glue.end([1])
    assert torch.equal(got[0], want[0].view(C, P, lat, 17, 3))
    assert got[1].cpu().numpy().reshape(C * P, lat).tolist() == want[1].tolist()
    assert got[2].cpu().numpy().reshape(-1).tolist() == want[2].tolist()
    assert (want[1][P:2 * P] >= 0).any() and (want[1][:P] < 0).all() and (want[1][2 * P:] < 0).all()


def test_one_person_equals_gen_pose():
    """one camera, one person present every tick, augment as gen_pose uses it, then end(): the final and tail poses
    are camera_to_world(evaluate_sequence(...)) placed frame by frame with that frame's keypoints"""
    T = 60
    model = _model('dilated', (3, 3, 3))
    lat = (model.receptive_field() - 1) // 2
    det, pose = _Darknet(1), _Pose().cuda()
    tick = LiveTick(det, pose, model, 1, (W, H), num_person=1, augment=True, graph=True, delayed=True)
    frames = torch.from_numpy(DR.synth_frames(1, H, W, seed=4)).cuda()
    poses, kpts = {}, []
    for t in range(T):
        x1, y1 = 30000 + 150 * t, 20000 + 40 * t
        det.preds.copy_(_predictions([np.array([[x1, y1, x1 + 25000, y1 + 60000]])], 900 + t))
        out = tick(frames)
        assert bool(out.active[0, 0]) and int(out.ids[0, 0]) == int(tick.out.ids[0, 0]) >= 1, t
        pid = int(out.ids[0, 0])
        kpts.append(out.keypoints[0, 0].clone())
        f = int(out.frame[0, 0])
        if f >= 0:
            poses[f] = out.poses[0, 0].clone()
    tail, tail_frame, tail_ids = tick.end()
    assert int(tail_ids[0, 0]) == pid and tail_frame[0, 0].tolist() == list(range(T - lat, T))
    for k in range(lat):
        poses[int(tail_frame[0, 0, k])] = tail[0, 0, k].clone()
    assert sorted(poses) == list(range(T))
    got = torch.stack([poses[f] for f in range(T)]).cpu().numpy()
    kp = torch.stack(kpts)
    x = Pp.normalize_screen(kp, W, H)
    y = tta.evaluate_sequence(model, x, [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16], [4, 5, 6, 11, 12, 13],
                              [1, 2, 3, 14, 15, 16])
    world = Pp.camera_to_world(y, LR.ROT, 0)
    want = torch.cat([DP.revise_skes_real_time(world[f:f + 1], kp[f:f + 1], W) for f in range(T)]).cpu().numpy()
    err = float(np.abs(got - want).max() / np.abs(want).max())
    assert err <= WHOLE_BAR, err


def test_two_runs_repeat_and_no_tick_synchronises():
    C, P, T = 3, 2, 40
    frames, ticks = _scene(C, T, seed=7)
    model = _model()
    runs = []
    for graph in (False, True, False):
        det, pose = _Darknet(C), _Pose().cuda()
        tick = LiveTick(det, pose, model, C, (W, H), num_person=P, augment=True, graph=graph, lookahead=0, max_gap=2,
                        delayed=True)
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
        assert tick.last_launches >= 15
    for r in runs[1:]:
        assert all(torch.equal(x, y) for a, b in zip(runs[0], r) for x, y in zip(a, b))


@pytest.mark.parametrize('graph', [False, True])
def test_stream_order(graph):
    C, P = 2, 2
    frames, ticks = _scene(C, 20, seed=11)
    model = _model()
    want = []
    for side in (False, True):
        det, pose = _Darknet(C), _Pose().cuda()
        tick = LiveTick(det, pose, model, C, (W, H), num_person=P, graph=graph, lookahead=0, delayed=True)
        for t in range(19):
            det.preds.copy_(ticks[t])
            tick(frames)
        torch.cuda.synchronize()
        if not side:
            det.preds.copy_(ticks[19])
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
            det.preds.copy_(ticks[19])
            out = tick(frames)
            assert not s.query(), 'synchronised with the host'
        s.synchronize()
        got = [x.cpu() for x in _snapshot(out)]
        assert all(torch.equal(x, y) for x, y in zip(got, want))


def test_refusals_come_before_any_launch_and_weights_follow_the_rule():
    C, P = 2, 2
    frames, ticks = _scene(C, 3, seed=5)
    det, pose = _Darknet(C), _Pose().cuda()
    m = _model()
    for kw in (dict(lookahead=13), dict(lookahead=-1), dict(max_gap=-1)):
        with pytest.raises(GastError, match='lookahead|max_gap'):
            LiveTick(det, pose, m, C, (W, H), delayed=True, **kw)
    causal = SpatioTemporalModelOptimized1f(adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], [])), 17, 2,
                                            17, [3, 3, 3], causal=True, channels=32).cuda().eval()
    with pytest.raises(GastError, match='delayed=True'):
        LiveTick(det, pose, m, C, (W, H), lookahead=0)      # the delayed tick is asked for by name
    for kw in (dict(lookahead=0), dict(max_gap=3), dict(delayed=True)):
        with pytest.raises(GastError, match='non-causal'):
            LiveTick(det, pose, causal, C, (W, H), **kw)
    with pytest.raises(GastError, match='causal tick'):
        LiveTick(det, pose, causal, C, (W, H)).end()
    dense = SpatioTemporalModel(adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], [])), 17, 2, 17,
                                [3, 3, 3], channels=32, dense=True).cuda().eval()
    with pytest.raises(GastError, match='dense'):
        LiveTick(det, pose, dense, C, (W, H), delayed=True)
    for graph in (False, True):
        tick = LiveTick(det, pose, m, C, (W, H), num_person=P, graph=graph, lookahead=0, delayed=True)
        assert tick.latency == 13
        det.preds.copy_(ticks[0])
        tick(frames)
        torch.cuda.synchronize()
        before = tick._status.clone()
        for bad in (frames[:1], frames.float(), frames.cpu()):
            with pytest.raises(GastError, match='frames'):
                tick(bad)
        with pytest.raises(GastError):
            tick.end([C])
        m.train()
        with pytest.raises(GastError, match='eval'):
            tick(frames)
        m.eval()
        with torch.no_grad():
            next(m.parameters()).mul_(1.0001)
        with pytest.raises(GastError, match='reset'):
            tick(frames)
        with pytest.raises(GastError, match='reset'):
            tick.end()
        assert torch.equal(tick._status, before)
        tick.reset()
        det.preds.copy_(ticks[1])
        tick(frames)
        assert int(tick._status[0, 1]) == 2
