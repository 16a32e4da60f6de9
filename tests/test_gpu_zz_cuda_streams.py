"""Every device call against torch's CUDA-stream contract: a call orders all of its work on the caller's current
stream, keeps no device buffer that another stream or a captured CUDA graph may still use, and so gives the same bits
on any stream, with other calls in flight, and when a user captures it in torch.cuda.graph.

  A. Stream order.  Each public entry runs once on the default stream and once on a fresh side stream behind a
     device sleep, with every device tensor it reads (inputs, and the model's parameters) NaN (integers 0) until the
     sleep ends.  Work that is not ordered on the side stream reads the poison whatever the timing, so the two results
     must be equal bit for bit.  Entries that make no host synchronisation must also return while the stream sleeps.
  B. Two streams and the caching allocator: a forward queued on one stream while a larger call on another grows what
     used to be a cached workspace, and a tensor allocated right after takes the freed block.
  C. A user's graph capture of model(x) and of run_model_mpjpe, replayed after a larger eager call.
  D. Two mpjpe forwards of one handle in flight on two streams, each with its own workspace, and two calls each of
     pipeline.mpjpe, revise_skes, revise_skes_real_time and pose_metrics in flight on two streams.

The default-stream results are held to fp64 or to the reference by the other test files; here only the stream changes.
"""
import copy
import ctypes as C
import functools
import time

import numpy as np
import pytest
import torch

from gast_b200 import engine, synth
from gast_b200 import pipeline as P

pytestmark = pytest.mark.gpu

SLEEP_MS = 50
J = 17
LEFT, RIGHT = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]

# every public entry that part A runs; test_zz_every_entry_ran holds the file to this list
ENTRIES = [
    'forward_fp32', 'forward_tf32', 'forward_fp16', 'forward_half', 'run_model_mpjpe', 'run_model_chunked',
    'eval_backward', 'eval_backward_chunked', 'train_dropout', 'block', 'local', 'multi_global',
    'causal_push', 'delayed_push_flush', 'stream_chunk', 'stream_peek', 'stream_subset', 'graphed_tick', 'stream_move',
    'mpjpe', 'p_mpjpe', 'adam_step', 'chunk_gather', 'camera', 'normalize_screen', 'revise_kpts', 'revise_skes',
    'h36m_coco_format', 'evaluate_sequences', 'epoch_trainer', 'dataset_prepare', 'render_frames', 'crop_persons',
    'decode_heatmaps', 'letterbox', 'person_boxes', 'video_boxes_keypoints',
]
RAN = set()


@functools.lru_cache(maxsize=None)
def _cycles_per_ms():
    """the spin count of torch.cuda._sleep per millisecond, measured on the device clock"""
    n = 20_000_000
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(1000)
    e0.record()
    torch.cuda._sleep(n)
    e1.record()
    e1.synchronize()
    return n / e0.elapsed_time(e1)


def _sleep(ms=SLEEP_MS):
    torch.cuda._sleep(int(_cycles_per_ms() * ms))


def _poison_(t):
    with torch.no_grad():
        t.fill_(float('nan') if t.is_floating_point() else 0)


def _flat(x, out):
    """the tensors, arrays and numbers of a result, in order"""
    if isinstance(x, torch.Tensor):
        out.append(x.detach().cpu().contiguous().numpy())
    elif isinstance(x, np.ndarray):
        out.append(np.ascontiguousarray(x))
    elif isinstance(x, (list, tuple)):
        for v in x:
            _flat(v, out)
    elif isinstance(x, dict):
        for k in sorted(x, key=str):
            _flat(x[k], out)
    elif x is None or isinstance(x, (int, float, bool, str, np.generic)):
        out.append(np.asarray(x if x is not None else 'None'))
    else:
        raise TypeError('cannot compare %r' % type(x))
    return out


def _assert_bits(got, want, name):
    a, b = _flat(got, []), _flat(want, [])
    assert len(a) == len(b), name
    for i, (u, v) in enumerate(zip(a, b)):
        assert u.dtype == v.dtype and u.shape == v.shape, (name, i, u.dtype, v.dtype, u.shape, v.shape)
        assert u.tobytes() == v.tobytes(), (name, i)


def _ordered(name, make, run, nosync=False):
    """make() -> (obj, held): a fresh object of the entry and the device tensors it reads; run(obj) -> the result.
    Once on the default stream, once on a side stream with `held` poisoned until a sleep ends; equal bit for bit."""
    RAN.add(name)
    t0 = time.perf_counter()
    obj, _ = make()
    want = run(obj)
    torch.cuda.synchronize()
    # the side stream sleeps far longer than the host needs for the call, so `nosync` cannot see a slow host as a sync
    ms = max(SLEEP_MS, min(5000.0, 20e3 * (time.perf_counter() - t0))) if nosync else SLEEP_MS
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        obj, held = make()
        saved = [t.detach().clone() for t in held]
        for t in held:
            _poison_(t)
        _sleep(ms)
        with torch.no_grad():
            for t, v in zip(held, saved):
                t.copy_(v)
        got = run(obj)
        if nosync:
            assert not s.query(), '%s synchronised with the host' % name
    s.synchronize()
    _assert_bits(got, want, name)
    return got


# ---------------------------------------------------------------------------------------------------------------
# models
# ---------------------------------------------------------------------------------------------------------------
def _adj():
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), LEFT, RIGHT))


@functools.lru_cache(maxsize=None)
def _base(kind='dilated', causal=False, dropout=0.0, ch=32):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    cls = SpatioTemporalModelOptimized1f if kind == 'o1f' else SpatioTemporalModel
    m = cls(_adj(), J, 2, J, [3, 3, 3], causal=causal, dropout=dropout, channels=ch)
    synth.randomize_module(m, 3)
    return m.cuda().eval()


def _fresh(base):
    """a copy of `base` with handles of its own, made on the current stream, and its tensors"""
    m = copy.deepcopy(base)
    return m, [v for _, v in engine.named_tensors(m)]


def _x(B, T, seed=5, dtype=torch.float32):
    return torch.from_numpy(synth.synth_input(B, T, J, 2, seed=seed)).cuda().to(dtype)


def _model_entry(name, base, x, run):
    def make():
        m, held = _fresh(base)
        xx = x.clone()
        return (m, xx), held + [xx]
    return _ordered(name, make, lambda o: run(*o))


def _no_grad_forward(m, x):
    with torch.no_grad():
        return m(x)


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'fp16'])
def test_forward_is_ordered(precision):
    base = copy.deepcopy(_base())
    engine.set_precision(base, precision)
    _model_entry('forward_' + precision, base, _x(3, 31), _no_grad_forward)


def test_half_forward_is_ordered():
    base = copy.deepcopy(_base()).half()
    _model_entry('forward_half', base, _x(3, 31, dtype=torch.float16), _no_grad_forward)


def test_run_model_mpjpe_is_ordered():
    x = _x(4, 27)
    tgt = torch.from_numpy(synth.synth_target(4, J, seed=7)).cuda().reshape(4, 1, J, 3)

    def make():
        m, held = _fresh(_base())
        xx, tt = x.clone(), tgt.clone()
        return (m, xx, tt), held + [xx, tt]
    _ordered('run_model_mpjpe', make, lambda o: engine.run_model_mpjpe(*o))


def test_run_model_chunked_is_ordered():
    _model_entry('run_model_chunked', _base(), _x(2, 60), lambda m, x: _no_grad_forward(
        lambda v: engine.run_model_chunked(m, v, 7), x))


def _eval_backward(m, x, max_frames=None):
    xx = x.detach().requires_grad_(True)
    y = m(xx) if max_frames is None else engine.run_model_chunked(m, xx, max_frames)
    g = torch.linspace(-1, 1, y.numel(), device=y.device).reshape(y.shape)
    y.backward(g)
    return [y, xx.grad] + [p.grad for p in m.parameters()]


def test_eval_backward_is_ordered():
    _model_entry('eval_backward', _base(), _x(2, 33), _eval_backward)


def test_eval_backward_chunked_is_ordered():
    _model_entry('eval_backward_chunked', _base(), _x(2, 40), lambda m, x: _eval_backward(m, x, 5))


def test_training_with_dropout_is_ordered():
    """the same host seed gives the same dropout masks on the device: the output and every gradient of a train-mode
    step with dropout equal bit for bit only if every mask is too (tests/dropoutref.py restates them)"""
    base = copy.deepcopy(_base('o1f', dropout=0.25)).train()

    def run(m, x):
        torch.manual_seed(11)
        y = m(x)
        g = torch.linspace(-1, 1, y.numel(), device=y.device).reshape(y.shape)
        y.backward(g)
        return [y] + [p.grad for p in m.parameters()] + [v for k, v in m.state_dict().items() if 'running' in k]
    _model_entry('train_dropout', base, _x(8, 27), run)


def _sub(name, pick, shape):
    base = pick(_base())
    x = torch.from_numpy(np.random.RandomState(3).standard_normal(shape).astype(np.float32)).cuda()
    _model_entry(name, base, x, _no_grad_forward)


def test_block_is_ordered():
    _sub('block', lambda m: m.layers_graph_conv[0], (2, 32, 5, J))


def test_local_is_ordered():
    _sub('local', lambda m: m.layers_graph_conv[0].local_graph_layer, (2, 5, J, 32))


def test_multi_global_is_ordered():
    _sub('multi_global', lambda m: m.layers_graph_conv[0].global_graph_layer, (2, 5, J, 32))


# ---------------------------------------------------------------------------------------------------------------
# the pose streams
# ---------------------------------------------------------------------------------------------------------------
def _pool_entry(name, base, x, run, cls=None, **kw):
    from gast_b200.realtime import PoseStream
    cls = cls or PoseStream

    def make():
        m, held = _fresh(base)
        xx = x.clone()
        return (cls(m, x.shape[0], **kw), xx), held + [xx]
    return _ordered(name, make, lambda o: run(*o))


def test_causal_push_is_ordered():
    from gast_b200.realtime import CausalStream
    x = _x(3, 8)
    _pool_entry('causal_push', _base(causal=True), x,
                lambda cs, x: [cs.push(x[:, t]) for t in range(x.shape[1])], cls=CausalStream)


def test_delayed_push_and_flush_are_ordered():
    def run(ps, x):
        out = [ps.push(x[:, t]) for t in range(x.shape[1])]
        ps.end()
        return out + [ps.push(x[:, 0]) for _ in range(ps.latency)]
    _pool_entry('delayed_push_flush', _base(), _x(2, 16), run)


def test_chunk_is_ordered():
    _pool_entry('stream_chunk', _base(), _x(3, 20), lambda ps, x: [ps.push_frames(x[:, :9]), ps.push_frames(x[:, 9:])],
                augment=True)


def test_peek_is_ordered():
    _pool_entry('stream_peek', _base(), _x(2, 10), lambda ps, x: [ps.push_frames(x), ps.peek(4)])


def test_subset_is_ordered():
    def run(ps, x):
        return [ps.push_frames(x[:, :6]), ps.push_frames(x[[2, 0], 6:9].contiguous(), streams=[2, 0]),
                ps.peek(3, streams=[0, 1])]
    _pool_entry('stream_subset', _base(), _x(3, 9), run)


def test_graphed_tick_is_ordered():
    from gast_b200.realtime import GraphedPoseStream

    def run(g, x):
        return [[t.clone() if isinstance(t, torch.Tensor) else t for t in g.push(x[:, k:k + 1])]
                for k in range(x.shape[1])]
    _pool_entry('graphed_tick', _base(), _x(2, 4), run, cls=GraphedPoseStream, peek=2)


def test_move_between_pools_is_ordered():
    from gast_b200.realtime import PoseStream

    def run(a, x):
        a.push_frames(x[:, :5])
        b = PoseStream(a.model, 2)
        b.push_frames(x[:2, :5])                       # an import keeps the pool's count: both pools at frame 5
        b.import_streams(a.export_streams([2, 0]), [1, 0])
        return b.push_frames(x[[0, 2], 5:].contiguous())
    _pool_entry('stream_move', _base(), _x(3, 8), run)


# ---------------------------------------------------------------------------------------------------------------
# gast_b200.pipeline
# ---------------------------------------------------------------------------------------------------------------
def _rand(*shape, seed=0, scale=1.0):
    return torch.from_numpy((scale * np.random.RandomState(seed).standard_normal(shape)).astype(np.float32)).cuda()


def _tensor_entry(name, fn, *args, nosync=False):
    """an entry of CUDA tensor arguments (anything else passes through unchanged)"""
    def make():
        a = [v.clone() if isinstance(v, torch.Tensor) else v for v in args]
        return a, [v for v in a if isinstance(v, torch.Tensor)]
    return _ordered(name, make, lambda a: fn(*a), nosync=nosync)


def test_mpjpe_is_ordered():
    def run(p, t):
        pp = p.detach().requires_grad_(True)
        loss = P.mpjpe(pp, t)
        (2.0 * loss).backward()
        return loss, pp.grad
    _tensor_entry('mpjpe', run, _rand(700, J, 3, seed=1), _rand(700, J, 3, seed=2))


def test_p_mpjpe_is_ordered():
    _tensor_entry('p_mpjpe', P.p_mpjpe_per_frame, _rand(300, J, 3, seed=3), _rand(300, J, 3, seed=4))


def test_adam_step_is_ordered():
    def run(p0, p1, g0, g1):
        ps = [torch.nn.Parameter(p0), torch.nn.Parameter(p1)]
        opt = P.FusedAdam(ps, lr=1e-3, amsgrad=True)
        out = []
        for k in range(3):
            ps[0].grad, ps[1].grad = g0 * (k + 1), g1 - k
            opt.step()
            out += [p.detach().clone() for p in ps]
        return out + [opt.exp_avg, opt.exp_avg_sq, opt.max_exp_avg_sq]
    _tensor_entry('adam_step', run, _rand(5000, seed=5), _rand(33, 7, seed=6), _rand(5000, seed=7),
                  _rand(33, 7, seed=8))


def test_chunk_gather_is_ordered():
    lens = [40, 23, 57]
    pairs = np.array([[s, a, a + 1, f] for s in range(3) for a, f in ((0, 0), (lens[s] - 1, 1), (lens[s] // 2, 1))])

    def run(a0, a1, a2, b0, b1, b2):
        seqs = P.DeviceSequences([a0, a1, a2], [b0, b1, b2])
        return P.chunk_gather(seqs, pairs, 1, 13, 0, LEFT, RIGHT, LEFT, RIGHT)
    _tensor_entry('chunk_gather', run, *[_rand(n, J, 2, seed=10 + i) for i, n in enumerate(lens)],
                  *[_rand(n, J, 3, seed=20 + i) for i, n in enumerate(lens)])


def test_camera_functions_are_ordered():
    q = np.array([0.5, -0.5, 0.5, 0.5], np.float32) / np.float32(1.0)
    t = np.array([0.3, -1.0, 4.0], np.float32)

    def run(x, seg, intr, g):
        w = P.camera_to_world(x, q, t)
        c = P.world_to_camera(w, q, t)
        return [w, c, P.project_to_2d_segments(x, seg, intr), P.project_to_2d_segments(x, seg, intr, grad_out=g)]
    x = _rand(50, J, 3, seed=11) + torch.tensor([0.0, 0.0, 5.0], device='cuda')
    seg = torch.tensor([0, 300, 50 * J], dtype=torch.int64, device='cuda')
    intr = torch.from_numpy(np.array([[1.1, 1.2, 0.01, -0.02, 0.1, -0.05, 0.01, 0.001, -0.002],
                                      [0.9, 1.0, -0.01, 0.02, -0.1, 0.05, 0.0, 0.002, 0.001]], np.float32)).cuda()
    _tensor_entry('camera', run, x, seg, intr, _rand(50, J, 2, seed=12))


def test_normalize_screen_is_ordered():
    _tensor_entry('normalize_screen', lambda x: [P.normalize_screen(x, 1920, 1080),
                                                 P.normalize_screen(x, 1000, 1002, inverse=True)],
                  _rand(40, J, 2, seed=13, scale=500.0))


def _person_slots(Pn=2, T=12, seed=14):
    rs = np.random.RandomState(seed)
    k = torch.from_numpy(rs.uniform(0, 1000, (Pn, T, 17, 2)).astype(np.float32)).cuda()
    s = torch.from_numpy(rs.uniform(0, 1, (Pn, T, 17)).astype(np.float32)).cuda()
    return k, s


def test_h36m_coco_format_is_ordered():
    _tensor_entry('h36m_coco_format', P.h36m_coco_format, *_person_slots())


def test_revise_kpts_is_ordered():
    k, s = _person_slots(seed=15)
    valid = torch.from_numpy(np.random.RandomState(16).randint(0, 2, (2, 12)).astype(np.int32)).cuda()
    _tensor_entry('revise_kpts', P.revise_kpts, k, s, valid, nosync=True)


def test_revise_skes_is_ordered():
    k, _ = _person_slots(seed=17)
    pred = _rand(20, 17, 3, seed=18)
    frames = torch.tensor(list(range(0, 10)) + list(range(2, 12)), dtype=torch.int64, device='cuda')
    _tensor_entry('revise_skes', lambda p, f, kk: P.revise_skes(p, f, [0, 10, 20], kk), pred, frames, k, nosync=True)


# ---------------------------------------------------------------------------------------------------------------
# evaluation, training and dataset preparation
# ---------------------------------------------------------------------------------------------------------------
def test_evaluate_sequences_is_ordered():
    from gast_b200.evaluation import evaluate_sequences
    lens = [40, 31, 60]
    p2 = [_rand(n, J, 2, seed=30 + i, scale=0.5) for i, n in enumerate(lens)]
    p3 = [_rand(n, J, 3, seed=40 + i, scale=0.3) for i, n in enumerate(lens)]
    groups = ['Walk', 'Sit', 'Walk']

    def run(m, *seqs):
        r = evaluate_sequences(m, list(seqs[:3]), list(seqs[3:]), groups, augment=True, kps_left=LEFT,
                               kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT, thresholds=True, n_streams=2,
                               chunk=32)
        return [[r[g].frames, r[g].mpjpe, r[g].p_mpjpe, r[g].pck, r[g].auc, r[g].per_joint] for g in r.groups]

    def make():
        m, held = _fresh(_base())
        seqs = [v.clone() for v in p2 + p3]
        return [m] + seqs, held + seqs
    _ordered('evaluate_sequences', make, lambda a: run(*a))


def test_epoch_trainer_is_ordered():
    """one epoch of EpochTrainer; its construction captures graphs (which synchronises), so the trainer is built
    first and the model's parameters are poisoned for the epoch"""
    from gast_b200 import training
    from device.common.generators import ChunkedGenerator
    rs = np.random.RandomState(21)
    lens = [30, 41, 25]
    p2 = [(0.5 * rs.standard_normal((n, J, 2))).astype(np.float32) for n in lens]
    p3 = [(0.3 * rs.standard_normal((n, J, 3))).astype(np.float32) for n in lens]
    base = copy.deepcopy(_base('o1f', dropout=0.1)).train()

    def build():
        m = copy.deepcopy(base)
        gen = ChunkedGenerator(40, None, p3, p2, 1, pad=13, causal_shift=0, shuffle=True, random_seed=1234,
                               augment=True, kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
        opt = P.FusedAdam(m.parameters(), lr=1e-3, amsgrad=True)
        return training.EpochTrainer(m, gen, opt), m, opt

    def run(o):
        tr, m, opt = o
        s, losses = tr.train_epoch_async()
        return [s, losses, opt.exp_avg, opt.exp_avg_sq] + [v for _, v in engine.named_tensors(m)]

    o = build()
    t0 = time.perf_counter()
    want = run(o)
    torch.cuda.synchronize()
    ms = max(SLEEP_MS, min(5000.0, 20e3 * (time.perf_counter() - t0)))
    RAN.add('epoch_trainer')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        o = build()
        torch.cuda.synchronize()
        held = [p for p in o[1].parameters()]
        saved = [t.detach().clone() for t in held]
        for t in held:
            _poison_(t)
        _sleep(ms)
        with torch.no_grad():
            for t, v in zip(held, saved):
                t.copy_(v)
        got = run(o)
        assert not s.query(), 'train_epoch_async synchronised with the host'
    s.synchronize()
    _assert_bits(got, want, 'epoch_trainer')


def test_dataset_preparation_is_ordered():
    """host arrays in: every upload and launch of prepare and fetch queues behind the sleep"""
    from gast_b200 import dataset as D
    from test_gpu_zz_dataset import _standin
    ds_in, pos2d, _, _ = _standin('h36m')

    def run(_):
        ds = D.prepare(ds_in, pos2d)
        return [ds.fetch(['S1'], ['Walk'], 5), ds.test_set(['S9', 'S1'], by_subject=True),
                ds.ground_truth_2d().fetch(['S9'], None, 1)]
    _ordered('dataset_prepare', lambda: (None, []), run, nosync=True)


# ---------------------------------------------------------------------------------------------------------------
# the video front end
# ---------------------------------------------------------------------------------------------------------------
def test_render_frames_is_ordered():
    from gast_b200 import render as R
    from test_gpu_zz_render import _Skel, H36M, META, _keypoints, _poses
    rng = np.random.default_rng(8)
    video = torch.from_numpy(rng.integers(0, 256, (12, 36, 64, 3), dtype=np.uint8)).cuda()
    kp = torch.from_numpy(_keypoints(rng, 12, 1, 17, 64, 36)).cuda()
    pr, pg = torch.from_numpy(_poses(rng, 12, 17)).cuda(), torch.from_numpy(_poses(rng, 12, 17)).cuda()
    R.render_frames(kp, {'r': pr, 'g': pg}, _Skel(H36M), 70., (64, 36), size=0.64, input_frames=video,
                    keypoints_metadata=META)
    _tensor_entry('render_frames', lambda k, a, b, v: R.render_frames(
        k, {'r': a, 'g': b}, _Skel(H36M), 70., (64, 36), size=0.64, input_frames=v, downsample=2, input_video_skip=1,
        keypoints_metadata=META), kp, pr, pg, video, nosync=True)


@pytest.fixture(scope='module')
def kp_gold():
    import keypoints2dref as KR
    from conftest import load_golden
    g = load_golden('keypoints2d')
    m = g['meta']
    g['frames'] = KR.synth_frames(m['F'], m['H'], m['W'])
    return g


def test_crop_persons_is_ordered(kp_gold):
    from gast_b200 import keypoints2d as K
    g = kp_gold
    frames = torch.from_numpy(g['frames']).cuda()
    K.crop_persons(frames, g['box_frame'], g['fwd_small'], g['meta']['small'])
    _tensor_entry('crop_persons', lambda f: K.crop_persons(f, g['box_frame'], g['fwd_small'], g['meta']['small']),
                  frames, nosync=True)


def test_decode_heatmaps_is_ordered(kp_gold):
    import keypoints2dref as KR
    from gast_b200 import keypoints2d as K
    hm = torch.from_numpy(KR.synth_heatmaps(16, 17, 96, 72, seed=9)).cuda()
    K.decode_heatmaps(hm, kp_gold['inv_72x96'])
    _tensor_entry('decode_heatmaps', lambda h: K.decode_heatmaps(h, kp_gold['inv_72x96']), hm, nosync=True)


def test_letterbox_is_ordered():
    import detectionref as DR
    from gast_b200 import detection as Dt
    frames = torch.from_numpy(DR.synth_frames(3, 300, 500, seed=8)).cuda()
    Dt.letterbox(frames, 416)
    _tensor_entry('letterbox', lambda f: Dt.letterbox(f, 416), frames, nosync=True)


def test_person_boxes_are_ordered():
    import detectionref as DR
    from gast_b200 import detection as Dt
    pred = torch.from_numpy(np.stack([DR.many_candidates(416, n, seed=n, ties=True) for n in (8, 30, 60)])).cuda()
    sizes = torch.tensor([[500, 300], [1920, 1080], [641, 481]], dtype=torch.int32).cuda()
    Dt.person_boxes(pred, sizes, 416)
    _tensor_entry('person_boxes', lambda p, sz: Dt.person_boxes(p, sz, 416), pred, sizes, nosync=True)


def test_video_boxes_into_video_keypoints_is_ordered():
    from gast_b200 import detection as Dt
    from gast_b200 import keypoints2d as K
    from test_gpu_zz_detection import _clip, _StandInDarknet, _Recorder
    D, preds, frames = _clip()
    net = _StandInDarknet(preds)

    class _Pose(torch.nn.Module):
        def forward(self, x):
            return torch.nn.functional.avg_pool2d(x, 4)[:, :1].repeat(1, 17, 1, 1)

    def run(f):
        tracker = _Recorder()
        out = Dt.video_boxes(f, net, tracker, D)
        kp, sc = K.video_keypoints(f, out, _Pose(), 1)
        return [kp, sc, tracker.seen, [o for o in out if o is not None]]
    _tensor_entry('video_boxes_keypoints', run, torch.from_numpy(frames).cuda())


# ---------------------------------------------------------------------------------------------------------------
# B. two streams and the caching allocator
# ---------------------------------------------------------------------------------------------------------------
def _forward_bytes(m, x):
    """the workspace of the model forward m(x)"""
    h = engine.model_handle(m, x.device)
    B, T = int(x.shape[0]), int(x.shape[1])
    return int(h.lib.gast_workspace_bytes(h.h, B, T, engine._strided_now(m, T)))


@pytest.fixture
def ws_log(monkeypatch):
    """the workspace pointer of every gast_forward / gast_forward_mpjpe call, in call order"""
    from gast_b200 import _lib
    lib, log = _lib.load(), []
    for entry, at in (('gast_forward', 6), ('gast_forward_mpjpe', 8)):
        def logged(*a, _f=getattr(lib, entry), _at=at):
            log.append(a[_at].value)
            return _f(*a)
        monkeypatch.setattr(lib, entry, logged)
    return log


def _overlap(a, b, n):
    """whether [a, a + n) and [b, b + n) overlap"""
    return a < b + n and b < a + n


def _two_streams(m, x, x_big, nbytes, ws_log):
    """m(x) queued on a side stream behind a sleep while a twice larger call runs on the default stream, then a
    tensor of `nbytes` (the size of m(x)'s workspace) is allocated and filled there.  The tensor must not overlap the
    workspace the queued forward writes (with one workspace kept per handle the larger call freed it and the tensor
    took it), must keep its pattern, and the queued forward must give the default-stream bits."""
    with torch.no_grad():
        del ws_log[:]
        want = m(x).clone()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _sleep()
            y1 = m(x)
        queued = ws_log[-1]
        m(x_big)
        z = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
    assert not _overlap(z.data_ptr(), queued, nbytes), 'a freed workspace was still in use by a queued forward'
    assert bool((z == 0xA5).all()), 'a forward queued on another stream wrote into a freed workspace'
    _assert_bits(y1, want, 'forward on a side stream')


def test_queued_forward_keeps_its_workspace_when_another_stream_grows(ws_log):
    m = copy.deepcopy(_base())
    x, x_big = _x(64, 27), _x(128, 27, seed=6)
    nbytes = _forward_bytes(m, x)
    assert nbytes > 10 << 20
    _two_streams(m, x, x_big, nbytes, ws_log)


def test_queued_sub_module_forward_keeps_its_workspace_when_another_stream_grows(ws_log):
    """a GraphAttentionBlock, whose forward writes every buffer of its workspace"""
    blk = copy.deepcopy(_base().layers_graph_conv[0])
    x = _rand(400, 32, 3, J, seed=22)
    x_big = _rand(800, 32, 3, J, seed=23)
    with torch.no_grad():
        blk(x)
    h = next(iter(blk.__dict__['_gast_handles'].values()))
    nbytes = int(h.lib.gast_workspace_bytes(h.h, 400 * 3, 1, 0))
    assert nbytes > 10 << 20
    _two_streams(blk, x, x_big, nbytes, ws_log)


# ---------------------------------------------------------------------------------------------------------------
# C. a user's CUDA graph capture
# ---------------------------------------------------------------------------------------------------------------
def _capture(fn):
    """torch's documented pattern: warm up on a side stream, then capture"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(g):
        out = fn()
    return g, out


def _replay_after_growth(m, fn, x_big, nbytes, name, ws_log):
    """capture fn(), make an eager call with twice the batch, allocate a filler of the size of fn's workspace, replay.
    The filler must not overlap the workspace the graph baked in (with one workspace kept per handle the eager call
    freed it and the filler took it), must keep its pattern, and the replay must give the eager bits."""
    with torch.no_grad():
        del ws_log[:]
        want = fn()
        g, out = _capture(fn)
        captured = ws_log[-1]
        m(x_big)
        filler = torch.full((nbytes,), 0x5A, dtype=torch.uint8, device='cuda')
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
    assert not _overlap(filler.data_ptr(), captured, nbytes), 'a freed workspace was still baked into a graph'
    assert bool((filler == 0x5A).all()), '%s: the graph replay wrote into memory it does not own' % name
    _assert_bits(out, want, name)


def test_captured_forward_replays_after_a_larger_eager_call(ws_log):
    m = copy.deepcopy(_base())
    x, x_big = _x(80, 27), _x(160, 27, seed=6)
    nbytes = _forward_bytes(m, x)
    assert nbytes > 10 << 20
    _replay_after_growth(m, lambda: m(x), x_big, nbytes, 'model(x)', ws_log)


def test_captured_run_model_mpjpe_replays_after_a_larger_eager_call(ws_log):
    m = copy.deepcopy(_base())
    x, x_big = _x(80, 27), _x(160, 27, seed=6)
    tgt = torch.from_numpy(synth.synth_target(80, J, seed=7)).cuda().reshape(80, 1, J, 3)
    nbytes = _forward_bytes(m, x)
    assert nbytes > 10 << 20
    _replay_after_growth(m, lambda: engine.run_model_mpjpe(m, x, tgt), x_big, nbytes, 'run_model_mpjpe', ws_log)


# ---------------------------------------------------------------------------------------------------------------
# D. two mpjpe forwards of one handle in flight
# ---------------------------------------------------------------------------------------------------------------
def test_two_mpjpe_calls_in_flight_on_one_handle():
    """both calls are released together by one event; each has its own workspace, so each loss is its own.  Overlap
    cannot be forced: this pins that the handle holds no per-call scratch (the partials and ticket of the loss are in
    the caller's workspace)."""
    m = copy.deepcopy(_base('o1f'))
    B, T = 64, 27
    xs = [_x(B, T, seed=31), _x(B, T, seed=32)]
    ts = [torch.from_numpy(synth.synth_target(B, J, seed=s)).cuda().reshape(B, 1, J, 3) for s in (33, 34)]
    want = [engine.run_model_mpjpe(m, x, t)[1].clone() for x, t in zip(xs, ts)]
    h = engine.model_handle(m, xs[0].device)
    sn = engine._strided_now(m, T)
    nbytes = int(h.lib.gast_workspace_bytes(h.h, B, T, sn))
    gate = torch.cuda.Stream()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    ws = [torch.empty(nbytes, dtype=torch.uint8, device='cuda') for _ in streams]
    ys = [torch.empty((B, 1, J, 3), device='cuda') for _ in streams]
    losses = [torch.full((), float('nan'), device='cuda') for _ in streams]
    torch.cuda.synchronize()
    ev = torch.cuda.Event()
    with torch.cuda.stream(gate):
        _sleep()
        ev.record(gate)
    for k, s in enumerate(streams):
        s.wait_event(ev)
        rc = h.lib.gast_forward_mpjpe(h.h, engine._p(xs[k]), engine._p(ts[k]), engine._p(ys[k]), engine._p(losses[k]),
                                      B, T, sn, engine._p(ws[k]), nbytes, C.c_void_p(s.cuda_stream))
        assert rc == 0
    torch.cuda.synchronize()
    for k in range(2):
        _assert_bits(losses[k], want[k], 'mpjpe on stream %d' % k)


def test_two_pipeline_mpjpe_calls_in_flight():
    """pipeline.mpjpe's block partials are the call's own: two losses released together on two streams are each their
    single-stream value (a scratch kept per device was shared by both)"""
    preds = [_rand(60000, J, 3, seed=51), _rand(60000, J, 3, seed=52)]
    tgts = [_rand(60000, J, 3, seed=53), _rand(60000, J, 3, seed=54)]
    want = [P.mpjpe(p, t).clone() for p, t in zip(preds, tgts)]
    torch.cuda.synchronize()
    gate, streams = torch.cuda.Stream(), [torch.cuda.Stream(), torch.cuda.Stream()]
    ev = torch.cuda.Event()
    with torch.cuda.stream(gate):
        _sleep()
        ev.record(gate)
    got = []
    for k, s in enumerate(streams):
        s.wait_event(ev)
        with torch.cuda.stream(s):
            got.append(P.mpjpe(preds[k], tgts[k]))
    torch.cuda.synchronize()
    for k in range(2):
        _assert_bits(got[k], want[k], 'pipeline.mpjpe on stream %d' % k)


def _prep_case(kind, seed):
    """inputs of revise_skes, revise_skes_real_time or pose_metrics, large enough that two calls overlap"""
    rs = np.random.RandomState(seed)
    if kind == 'revise_skes':
        Pn, T = 4, 3000
        kp = torch.from_numpy(rs.uniform(0, 1000, (Pn, T, 17, 2)).astype(np.float32)).cuda()
        pred = _rand(Pn * T, 17, 3, seed=seed + 1)
        frames = torch.arange(T, device='cuda').repeat(Pn)
        return lambda: P.revise_skes(pred, frames, [k * T for k in range(Pn + 1)], kp)
    if kind == 'revise_skes_real_time':
        pred, kp = _rand(20000, 17, 3, seed=seed + 1), _rand(20000, 17, 2, seed=seed + 2, scale=500.0)
        return lambda: P.revise_skes_real_time(pred, kp, 1280)
    pred, tgt = _rand(200000, 17, 3, seed=seed + 1), _rand(200000, 17, 3, seed=seed + 2)
    seg = [0, 1000, 150000, 200000]
    return lambda: P.pose_metrics(pred, tgt, seg, thresholds=[0.5, 1.0], distances=True)


@pytest.mark.parametrize('kind', ['revise_skes', 'revise_skes_real_time', 'pose_metrics'])
def test_two_placement_or_metric_calls_in_flight(kind):
    """the scratch of revise_skes, revise_skes_real_time and pose_metrics is the call's own: two calls released together
    on two streams are each their single-stream value (a scratch kept per device was shared by both, and growing it
    freed it under a queued call)"""
    calls = [_prep_case(kind, 60), _prep_case(kind, 70)]
    want = [c() for c in calls]
    torch.cuda.synchronize()
    gate, streams = torch.cuda.Stream(), [torch.cuda.Stream(), torch.cuda.Stream()]
    ev = torch.cuda.Event()
    with torch.cuda.stream(gate):
        _sleep()
        ev.record(gate)
    got = []
    for c, s in zip(calls, streams):
        s.wait_event(ev)
        with torch.cuda.stream(s):
            got.append(c())
    torch.cuda.synchronize()
    for k in range(2):
        _assert_bits(got[k], want[k], '%s on stream %d' % (kind, k))


def _a_tests():
    """the names of this file's part A tests"""
    return {k for k, v in globals().items() if k.startswith('test_') and callable(v)
            and (k.endswith('_is_ordered') or k.endswith('_are_ordered'))}


def test_zz_every_entry_ran(request):
    """part A ran every public entry listed in ENTRIES, and ENTRIES lists every entry part A ran: a new entry point
    is added to both.  Skipped when this run did not collect every part A test (-k, a node id, --lf, xdist)."""
    here = {it.originalname for it in request.session.items if it.module is request.module}
    if not _a_tests() <= here or hasattr(request.config, 'workerinput'):
        pytest.skip('this run does not include every part A test')
    assert RAN == set(ENTRIES), (sorted(set(ENTRIES) - RAN), sorted(RAN - set(ENTRIES)))
