"""The video demo's keypoint repair and person placement on the device (device.tools.preprocess / device.tools.inference,
csrc/pipeline.cuh) against the unmodified reference's outputs (tests/golden/preprocess_17.npz) and the numpy oracle
(tests/preprocessref.py): bit for bit, except the lifting forward itself, which is held to the project's 1e-4."""
import numpy as np
import pytest
import torch

from conftest import load_golden
import preprocessref as R

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
    return load_golden('preprocess_17')


def _frames(G, name):
    return [G['%s_valid%d' % (name, p)] for p in range(int(G[name + '_n_person']))]


def _np(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def _same(a, b):
    a, b = _np(a), _np(b)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert a.dtype == b.dtype, (a.dtype, b.dtype)
    assert np.array_equal(a, b), np.nanmax(np.abs(a.astype(np.float64) - b))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _model(G, causal=False, strided=False):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from gast_b200 import synth
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    meta = G['meta']['gen_pose']
    adj = adj_mx_from_skeleton(Skeleton(parents=synth.skeleton_parents(17), joints_left=[], joints_right=[]))
    cls = SpatioTemporalModelOptimized1f if strided else SpatioTemporalModel
    m = cls(adj, 17, 2, 17, meta['filter_widths'], causal=causal, channels=meta['channels'], dropout=0.05)
    synth.randomize_module(m, meta['seed'])
    return m.cuda().eval()


@pytest.mark.parametrize('name', ['baseball', 'two'])
@pytest.mark.parametrize('on_dev', [False, True])
def test_h36m_coco_format_and_revise_kpts(G, name, on_dev):
    import device.tools.preprocess as D
    kp, sc = G[name + '_kp'], G[name + '_sc']
    hk, hs, vf = D.h36m_coco_format(_cuda(kp), _cuda(sc)) if on_dev else D.h36m_coco_format(kp, sc)
    for x in (hk, hs) + tuple(vf):
        assert isinstance(x, torch.Tensor if on_dev else np.ndarray) and (not on_dev or x.is_cuda)
    _same(hk, G[name + '_h36m_kpts'])
    _same(hs, G[name + '_h36m_scores'])
    ref = _frames(G, name)
    assert len(vf) == len(ref)
    for a, b in zip(vf, ref):
        _same(a, b)
    _same(D.revise_kpts(hk, hs, vf), G[name + '_re_kpts'])
    if on_dev:                                                # host frame lists with CUDA keypoints
        _same(D.revise_kpts(hk, hs, ref), G[name + '_re_kpts'])


@pytest.mark.parametrize('on_dev', [False, True])
def test_revise_kpts_rules_and_threshold(G, on_dev):
    import device.tools.preprocess as D
    k, s, v = G['rk_kpts'], G['rk_scores'], [G['rk_valid']]
    got = D.revise_kpts(_cuda(k), _cuda(s), [_cuda(v[0])]) if on_dev else D.revise_kpts(k, s, v)
    _same(got, G['rk_out'])


@pytest.mark.parametrize('n', [1, 2])
@pytest.mark.parametrize('frames_on_dev', [False, True])
def test_revise_skes(G, n, frames_on_dev):
    import device.tools.preprocess as D
    vf = [G['two_valid0'], G['two_valid1']][:n]
    pred = [G['skes%d_pred%d' % (n, p)] for p in range(n)]
    re = G['two_re_kpts'][:n]
    _same(D.revise_skes(pred, re, vf), G['skes%d_out' % n])
    got = D.revise_skes([_cuda(p) for p in pred], _cuda(re), [_cuda(f) for f in vf] if frames_on_dev else vf)
    assert got.is_cuda
    _same(got, G['skes%d_out' % n])


@pytest.mark.parametrize('M', [1, 2, 64])
@pytest.mark.parametrize('width', [1920, 1280])
def test_revise_skes_real_time(G, M, width):
    import device.tools.preprocess as D
    key = 'rt_M%d_w%d' % (M, width)
    _same(D.revise_skes_real_time(G[key + '_pred'], G[key + '_kpts'], width), G[key + '_out'])
    got = D.revise_skes_real_time(_cuda(G[key + '_pred']), _cuda(G[key + '_kpts']), width)
    assert got.is_cuda
    _same(got, G[key + '_out'])


def _big_offline(T, seed):
    """two persons over T frames: invalid stretches and holes, partly overlapping, scores spread around 0.3"""
    rs = np.random.RandomState(seed)
    kp = rs.uniform(0, 1900, (2, T, 17, 2)).astype(np.float32)
    sc = rs.uniform(0.0, 1.0, (2, T, 17)).astype(np.float32)
    sc[..., [2, 3, 5, 6]] = rs.uniform(0.2, 0.4, (2, T, 4)).astype(np.float32)
    for p, (lo, hi) in enumerate(((0, int(0.7 * T)), (int(0.3 * T), T))):
        kp[p, :lo] = 0
        kp[p, hi:] = 0
        holes = rs.randint(0, T, T // 50)
        kp[p, holes] = 0
    return kp, sc


def test_full_size_offline_chain_vs_oracle():
    """2 persons x 100k frames: h36m_coco_format -> revise_kpts -> revise_skes, the device chain equals the oracle"""
    import device.tools.preprocess as D
    T = 100_000
    kp, sc = _big_offline(T, 5)
    hk, hs, vf = R.h36m_coco_format(kp, sc)
    re = R.revise_kpts(hk, hs, vf)
    rs = np.random.RandomState(6)
    pred = [rs.standard_normal((len(f), 17, 3)).astype(np.float32) for f in vf]
    want = R.revise_skes(pred, re, vf)
    dk, ds, dvf = D.h36m_coco_format(_cuda(kp), _cuda(sc))
    _same(dk, hk)
    _same(ds, hs)
    for a, b in zip(dvf, vf):
        _same(a, b)
    dre = D.revise_kpts(dk, ds, dvf)
    _same(dre, re)
    got = D.revise_skes([_cuda(p) for p in pred], dre, dvf)
    _same(got, want)
    again = D.revise_skes([_cuda(p) for p in pred], dre, dvf)
    assert torch.equal(got, again)                   # repeatable bit for bit
    assert float(want[..., 2].min()) == 0.0 or np.isnan(want).any()


def test_full_size_real_time_vs_oracle():
    import device.tools.preprocess as D
    rs = np.random.RandomState(8)
    M = 4096
    pred = rs.standard_normal((M, 17, 3)).astype(np.float32)
    for width in (1920, 1280, 1000.5):
        k = rs.uniform(0, width, (M, 17, 2)).astype(np.float32)
        got = D.revise_skes_real_time(_cuda(pred), _cuda(k), width)
        _same(got, R.revise_skes_real_time(pred, k, width))
        assert torch.equal(got, D.revise_skes_real_time(_cuda(pred), _cuda(k), width))
    k3 = np.concatenate([k, rs.uniform(0, 1, (M, 17, 1)).astype(np.float32)], -1)     # (x, y, score) keypoints
    _same(D.revise_skes_real_time(_cuda(pred), _cuda(k3), 1000.5), R.revise_skes_real_time(pred, k3, 1000.5))


def test_errors(G):
    import device.tools.preprocess as D
    from gast_b200.engine import GastError
    with pytest.raises(RuntimeError, match='no CPU path'):
        D.revise_skes_real_time(torch.zeros(2, 17, 3), torch.zeros(2, 17, 2), 1920)
    with pytest.raises(RuntimeError, match='no CPU path'):
        D.h36m_coco_format(torch.zeros(2, 5, 17, 2), torch.zeros(2, 5, 17))
    with pytest.raises(RuntimeError, match='no CPU path'):
        D.revise_kpts(torch.zeros(1, 5, 17, 2), torch.zeros(1, 5, 17), [np.arange(5)])
    with pytest.raises(GastError, match='17 joints'):
        D.revise_skes_real_time(torch.zeros(2, 16, 3, device='cuda'), torch.zeros(2, 16, 2, device='cuda'), 1920)
    with pytest.raises(GastError, match='17 joints'):
        D.revise_skes_real_time(np.zeros((2, 19, 3), np.float32), np.zeros((2, 19, 2), np.float32), 1920)
    dk = G['disjoint_kpts']
    dp = [G['disjoint_pred0'], G['disjoint_pred1']]
    dv = [G['disjoint_valid0'], G['disjoint_valid1']]
    with pytest.raises(ValueError):
        D.revise_skes(dp, dk, dv)
    with pytest.raises(ValueError):
        D.revise_skes([_cuda(p) for p in dp], _cuda(dk), dv)
    # CUDA index tensors: no host read, so no exception; the two persons' x and y come out NaN
    got = D.revise_skes([_cuda(p) for p in dp], _cuda(dk), [_cuda(v) for v in dv]).cpu().numpy()
    for p in range(2):
        assert np.isnan(got[p, dv[p], :, :2]).all()


def test_no_host_sync_on_cuda_inputs(G):
    import device.tools.preprocess as D
    vf = [G['two_valid0'], G['two_valid1']]
    hk, hs, re = _cuda(G['two_h36m_kpts']), _cuda(G['two_h36m_scores']), _cuda(G['two_re_kpts'])
    dvf = [_cuda(f) for f in vf]
    pred = [_cuda(G['skes2_pred0']), _cuda(G['skes2_pred1'])]
    key = 'rt_M64_w1280'
    rp, rk = _cuda(G[key + '_pred']), _cuda(G[key + '_kpts'])
    for frames in (dvf, vf):
        D.revise_kpts(hk, hs, frames)
        D.revise_skes(pred, re, frames)            # warm-up: library load, workspace
    D.revise_skes_real_time(rp, rk, 1280)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        outs = []
        for frames in (dvf, vf):
            outs.append(D.revise_kpts(hk, hs, frames))
            outs.append(D.revise_skes(pred, re, frames))
        outs.append(D.revise_skes_real_time(rp, rk, 1280))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for o, want in zip(outs, ['two_re_kpts', 'skes2_out', 'two_re_kpts', 'skes2_out', key + '_out']):
        _same(o, G[want])


@pytest.mark.parametrize('name', ['baseball', 'two'])
@pytest.mark.parametrize('on_dev', [False, True])
def test_end_to_end_gen_pose_revise_skes(G, name, on_dev):
    """the demo's chain (gen_skes.py:115-134) on the device against the reference's, within the project's 1e-4"""
    import device.tools.preprocess as D
    import device.tools.inference as I
    m = _model(G)
    W, H, pad = G['meta']['width'], G['meta']['height'], G['meta']['gen_pose']['pad']
    kp, sc = G[name + '_kp'], G[name + '_sc']
    if on_dev:
        kp, sc = _cuda(kp), _cuda(sc)
    hk, hs, vf = D.h36m_coco_format(kp, sc)
    re = D.revise_kpts(hk, hs, vf)
    _same(re, G[name + '_re_kpts'])
    pred = I.gen_pose(re, vf, W, H, m, pad, 0)
    assert len(pred) == len(vf)
    for p, q in enumerate(pred):
        assert isinstance(q, torch.Tensor) == on_dev
        want = G['%s_pose%d' % (name, p)]
        assert _np(q).shape == want.shape
        assert np.abs(_np(q) - want).max() < 1e-4
    skes = D.revise_skes(pred, re, vf)
    assert isinstance(skes, torch.Tensor) == on_dev
    err = np.abs(_np(skes) - G[name + '_skes']).max()
    assert err < 1e-4, err


def test_inference_forms_agree(G):
    """evaluate / gen_pose_frame / gen_pose_frame_ against gen_pose and tta.evaluate_sequence on the same keypoints"""
    import device.tools.inference as I
    from device.common.generators import UnchunkedGenerator
    from gast_b200 import pipeline as P, tta
    m = _model(G)
    W, H, pad = G['meta']['width'], G['meta']['height'], G['meta']['gen_pose']['pad']
    re = _cuda(G['two_re_kpts'])
    f0 = _cuda(G['two_valid0'])
    seq = re[0].index_select(0, f0)
    norm = P.normalize_screen(seq, W, H)
    gen = UnchunkedGenerator(None, None, [norm.cpu().numpy()], pad=pad, causal_shift=0, augment=True, kps_left=I.kps_left,
                             kps_right=I.kps_right, joints_left=I.joints_left, joints_right=I.joints_right)
    ev = I.evaluate(gen, m)
    assert len(ev) == 1 and ev[0].is_cuda
    assert torch.equal(ev[0], tta.evaluate_sequence(m, norm, I.kps_left, I.kps_right, I.joints_left, I.joints_right))
    world = P.camera_to_world(ev[0], I.rot, 0)
    assert torch.equal(I.gen_pose(re[:1], [f0], W, H, m, pad, 0)[0], world)
    whole = I.gen_pose_frame_(seq, W, H, m, pad, 0)
    assert torch.equal(whole, world - torch.nn.functional.pad(world[..., 2:].amin().reshape(1), (2, 0)))
    win = seq[:2 * pad + 1]
    one = I.gen_pose_frame(torch.stack([win, win]), W, H, m, pad, 0)
    assert len(one) == 2 and one[0].shape == (17, 3) and torch.equal(one[0], one[1])
    w0 = P.camera_to_world(tta.evaluate_sequence(m, P.normalize_screen(win, W, H), I.kps_left, I.kps_right,
                                                 I.joints_left, I.joints_right), I.rot, 0)[0]
    assert np.abs(_np(one[0]) - _np(w0 - torch.nn.functional.pad(w0[:, 2:].amin().reshape(1), (2, 0)))).max() < 1e-5
    nb = I.gen_pose_frame(_np(torch.stack([win])), W, H, m, pad, 0)
    assert isinstance(nb[0], np.ndarray) and np.array_equal(nb[0], _np(one[0]))


def test_tick_loop_pose_stream(G):
    """a real-time loop: a causal 27-frame PoseStream with augmentation over 3 streams, each push's poses placed on
    the device; equal to the oracle on the same poses, bit for bit"""
    import device.tools.preprocess as D
    import device.tools.inference as I
    from gast_b200 import pipeline as P
    from gast_b200.realtime import PoseStream
    m = _model(G, causal=True, strided=True)
    ps = PoseStream(m, 3, augment=True, kps_left=I.kps_left, kps_right=I.kps_right, joints_left=I.joints_left,
                    joints_right=I.joints_right)
    rs = np.random.RandomState(12)
    walk = 900 + np.cumsum(rs.standard_normal((40, 3, 1, 2)) * 5, 0) + rs.uniform(-150, 150, (1, 3, 17, 2))
    pix = _cuda(walk.astype(np.float32))
    for t in range(40):
        poses, _ = ps.push(P.normalize_screen(pix[t], 1920, 1080))
        got = D.revise_skes_real_time(poses, pix[t], 1920)
        assert got.is_cuda and got.shape == (3, 17, 3)
        _same(got, R.revise_skes_real_time(_np(poses), _np(pix[t]), 1920))
