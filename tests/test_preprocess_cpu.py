"""CPU checks of the numpy restatement of the video demo's keypoint repair and person placement (tests/preprocessref.py)
against the unmodified reference's outputs (tests/golden/preprocess_17.npz): bit for bit."""
import numpy as np
import pytest

from conftest import load_golden
import preprocessref as R


@pytest.fixture(scope='module')
def G():
    return load_golden('preprocess_17')


def _frames(G, name):
    return [G['%s_valid%d' % (name, p)] for p in range(int(G[name + '_n_person']))]


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    assert np.array_equal(a, b), np.abs(a.astype(np.float64) - b).max()


@pytest.mark.parametrize('name', ['baseball', 'two'])
def test_h36m_coco_format_and_revise_kpts(G, name):
    hk, hs, vf = R.h36m_coco_format(G[name + '_kp'], G[name + '_sc'])
    _same(hk, G[name + '_h36m_kpts'])
    _same(hs, G[name + '_h36m_scores'])
    ref = _frames(G, name)
    assert len(vf) == len(ref) == (1 if name == 'baseball' else 2)     # baseball's empty second slot is dropped
    for a, b in zip(vf, ref):
        _same(a, b)
    _same(R.revise_kpts(hk, hs, vf), G[name + '_re_kpts'])


def test_revise_kpts_rules_and_threshold(G):
    _same(R.revise_kpts(G['rk_kpts'], G['rk_scores'], [G['rk_valid']]), G['rk_out'])
    changed = (G['rk_out'] != G['rk_kpts'])[0].any(axis=(1, 2))
    # frame t < 16 has low joints {(2, 3, 5, 6)[b] : bit b of t}: the six rules fire at 2, 8, 10, 11, 14, 15; frame 7
    # is not a valid frame and is zeroed; every other combination leaves the pose as it is
    assert sorted(np.nonzero(changed[:16])[0].tolist()) == [2, 7, 8, 10, 11, 14, 15]


@pytest.mark.parametrize('name', ['baseball', 'two'])
def test_chain_revise_skes(G, name):
    vf = _frames(G, name)
    _same(R.revise_skes([G['%s_pose%d' % (name, p)] for p in range(len(vf))], G[name + '_re_kpts'], vf),
          G[name + '_skes'])


@pytest.mark.parametrize('n', [1, 2])
def test_revise_skes(G, n):
    vf = [G['two_valid0'], G['two_valid1']][:n]
    _same(R.revise_skes([G['skes%d_pred%d' % (n, p)] for p in range(n)], G['two_re_kpts'][:n], vf), G['skes%d_out' % n])


def test_revise_skes_disjoint_raises(G):
    assert bool(G['disjoint_raises'])
    with pytest.raises(ValueError):
        R.revise_skes([G['disjoint_pred0'], G['disjoint_pred1']], G['disjoint_kpts'],
                      [G['disjoint_valid0'], G['disjoint_valid1']])


@pytest.mark.parametrize('M', [1, 2, 64])
@pytest.mark.parametrize('width', [1920, 1280])
def test_revise_skes_real_time(G, M, width):
    key = 'rt_M%d_w%d' % (M, width)
    _same(R.revise_skes_real_time(G[key + '_pred'], G[key + '_kpts'], width), G[key + '_out'])


def test_device_modules_keep_the_reference_names_and_refuse_cpu_tensors():
    import torch
    import device.tools.preprocess as D
    import device.tools.inference as I
    for n in ('h36m_coco_format', 'revise_kpts', 'load_kpts_json', 'revise_skes', 'revise_skes_real_time'):
        assert callable(getattr(D, n)), n
    for n in ('evaluate', 'gen_pose', 'gen_pose_frame', 'gen_pose_frame_'):
        assert callable(getattr(I, n)), n
    assert I.rot.dtype == np.float32 and I.rot.shape == (4,)
    assert I.joints_left == I.kps_left == [4, 5, 6, 11, 12, 13] and I.joints_right == I.kps_right == [1, 2, 3, 14, 15, 16]
    with pytest.raises(RuntimeError, match='no CPU path'):
        D.revise_skes_real_time(torch.zeros(2, 17, 3), torch.zeros(2, 17, 2), 1920)
    with pytest.raises(RuntimeError, match='no CPU path'):
        D.revise_kpts(torch.zeros(1, 4, 17, 2), torch.zeros(1, 4, 17), [np.arange(4)])
