"""The animation frames rendered on the device (gast_b200.render, csrc/render.cuh; DESIGN.md §8.5):
  * frames equal the numpy restatement (tests/renderref.py) bit for bit: one person on black, a background video of
    another size than the panel, two persons in a shared panel, two 3D panels (reconstruction and ground truth, also
    following the root as trainval.py --render does), downsample with limit and input_video_skip, 19-joint poses;
  * the device downsample equals the restatement, and so the reference's downsample_tensor, bit for bit;
  * several frame ranges give the bytes of one call, and two calls the same bytes;
  * render_frames makes no host synchronisation;
  * render_animation pipes exactly the frames to ffmpeg (a stub on PATH), and refuses without ffmpeg."""
import os
import stat

import numpy as np
import pytest
import torch

import renderref as RR
from gast_b200 import render as R
from gast_b200.engine import GastError

pytestmark = pytest.mark.gpu

H36M = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15]
H36M_TOE = H36M + [3, 6]                      # 19 joints: a toe under each ankle
RIGHT = [1, 2, 3, 14, 15, 16]
META = {'keypoints_symmetry': ([4, 5, 6, 11, 12, 13], RIGHT), 'layout_name': 'h36m'}


class _Skel(object):
    def __init__(self, parents):
        self._p = list(parents)

    def parents(self):
        return np.array(self._p)

    def joints_right(self):
        return RIGHT


def _poses(rng, T, J, x0=0., walk=0.):
    """a plausible skeleton wandering inside the axis box, one all-zero frame (an invalid frame of the demo)"""
    root = np.stack([x0 + walk * np.arange(T), 0.1 * np.sin(np.arange(T)), 0.9 + 0.05 * np.cos(np.arange(T))], 1)
    p = root[:, None, :] + rng.normal(0, 0.35, (T, J, 3))
    p[:, 0] = root
    p[min(2, T - 1)] = 0
    return p.astype(np.float32)


def _keypoints(rng, T, M, J, w, h):
    k = np.stack([rng.uniform(-0.05 * w, 1.05 * w, (T, M, J)), rng.uniform(-0.05 * h, 1.05 * h, (T, M, J))], -1)
    return k.astype(np.float32)


def _expected(kp, poses, skel, azim, viewport, size, input_frames=None, com=False, limit=-1, factor=1, skip=0,
              follow_root=False, bones_2d=None, frames=None):
    k, p, v, n = RR.scene(kp, poses, input_frames, limit, factor, skip)
    M, J = k.shape[1], k.shape[2]
    S = R.panel_side(size, 100)
    shared = com and M == 2
    H, W = (input_frames.shape[1], input_frames.shape[2]) if input_frames is not None else (viewport[1], viewport[0])
    geo = R.geometry(S, 100, H, W, azim, shared)
    flags = (RR.SHARED_PANEL if shared else 0) | (RR.FOLLOW_ROOT if follow_root else 0) | \
            (RR.BONES_2D if (J == 17 if bones_2d is None else bones_2d) else 0)
    frames = list(range(n)) if frames is None else list(frames)
    return RR.render(k, p, v, H, W, np.array(skel.parents()), R.color_table(J), RIGHT, min(J, 17), S, geo, flags, frames)


def _same(got, want):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else got
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = got != want
    assert not bad.any(), '%d of %d bytes differ, max |diff| %d' % (
        bad.sum(), bad.size, np.abs(got.astype(int) - want.astype(int)).max())


def test_one_person_on_black():
    rng = np.random.default_rng(0)
    kp, ps = _keypoints(rng, 7, 1, 17, 160, 120), [_poses(rng, 7, 17)]
    sk = _Skel(H36M)
    got = R.render_frames(kp, {'Reconstruction': ps[0]}, sk, 70., (160, 120), size=0.64, keypoints_metadata=META)
    assert got.is_cuda and got.dtype == torch.uint8 and tuple(got.shape) == (7, 64, 128, 3)
    _same(got, _expected(kp, ps, sk, 70., (160, 120), 0.64))


def test_background_video_of_another_size():
    rng = np.random.default_rng(1)
    video = rng.integers(0, 256, (6, 45, 80, 3), dtype=np.uint8)
    kp, ps = _keypoints(rng, 6, 1, 17, 80, 45), [_poses(rng, 6, 17)]
    sk = _Skel(H36M)
    got = R.render_frames(torch.from_numpy(kp).cuda(), [torch.from_numpy(ps[0]).cuda()], sk, -35., (80, 45), size=0.96,
                          input_frames=torch.from_numpy(video).cuda(), keypoints_metadata=META)
    _same(got, _expected(kp, ps, sk, -35., (80, 45), 0.96, input_frames=video))
    tall = rng.integers(0, 256, (6, 90, 40, 3), dtype=np.uint8)           # taller than wide, larger than the panel
    got = R.render_frames(kp, ps, sk, 10., (40, 90), size=0.64, input_frames=tall, keypoints_metadata=META)
    _same(got, _expected(kp, ps, sk, 10., (40, 90), 0.64, input_frames=tall))


def test_two_persons_in_a_shared_panel():
    rng = np.random.default_rng(2)
    kp = _keypoints(rng, 5, 2, 17, 120, 120)
    ps = [_poses(rng, 5, 17, x0=-0.9), _poses(rng, 5, 17, x0=0.9)]
    sk = _Skel(H36M)
    got = R.render_frames(kp, {'Reconstruction 1': ps[0], 'Reconstruction 2': ps[1]}, sk, 70., (120, 120), size=0.8,
                          com_reconstrcution=True, keypoints_metadata=META)
    assert tuple(got.shape) == (5, 80, 160, 3)
    _same(got, _expected(kp, ps, sk, 70., (120, 120), 0.8, com=True))


@pytest.mark.parametrize('follow_root', [False, True])
def test_reconstruction_and_ground_truth_panels(follow_root):
    rng = np.random.default_rng(3)
    kp = _keypoints(rng, 6, 1, 17, 100, 100)[:, 0]                         # visualization.py's (T, J, 2)
    ps = [_poses(rng, 6, 17, walk=0.3), _poses(rng, 6, 17, walk=0.3)]
    sk = _Skel(H36M)
    got = R.render_frames(kp, {'Reconstruction': ps[0], 'Ground truth': ps[1]}, sk, 45., (100, 100), size=0.64,
                          follow_root=follow_root, keypoints_metadata=META)
    assert tuple(got.shape) == (6, 64, 192, 3)
    _same(got, _expected(kp, ps, sk, 45., (100, 100), 0.64, follow_root=follow_root))


@pytest.mark.parametrize('factor,limit,skip', [(3, -1, 0), (2, 5, 0), (1, 12, 3), (3, 16, 2), (2, -1, 4)])
def test_downsample_limit_and_skip(factor, limit, skip):
    rng = np.random.default_rng(4 + factor + skip)
    T = 20
    video = rng.integers(0, 256, (T + 3, 30, 50, 3), dtype=np.uint8)
    kp, ps = _keypoints(rng, T, 1, 17, 50, 30), [_poses(rng, T, 17), _poses(rng, T - 1, 17)]
    sk = _Skel(H36M)
    got = R.render_frames(kp, ps, sk, 70., (50, 30), size=0.64, input_frames=video, limit=limit, downsample=factor,
                          input_video_skip=skip, keypoints_metadata=META)
    want = _expected(kp, ps, sk, 70., (50, 30), 0.64, input_frames=video, limit=limit, factor=factor, skip=skip)
    assert len(want) > 0
    _same(got, want)
    # without a video: a black image, no skip
    got = R.render_frames(kp, ps, sk, 70., (50, 30), size=0.64, limit=limit, downsample=factor, input_video_skip=skip,
                          keypoints_metadata=META)
    _same(got, _expected(kp, ps, sk, 70., (50, 30), 0.64, limit=limit, factor=factor))


def test_nineteen_joint_poses():
    rng = np.random.default_rng(5)
    kp, ps = _keypoints(rng, 4, 1, 19, 64, 64), [_poses(rng, 4, 19)]
    sk = _Skel(H36M_TOE)
    got = R.render_frames(kp, ps, sk, 70., (64, 64), size=0.64, keypoints_metadata=META)
    _same(got, _expected(kp, ps, sk, 70., (64, 64), 0.64))
    with_bones = R.Scene(kp, ps, sk, 70., (64, 64), size=0.64, keypoints_metadata=META, bones_2d=True).render()
    _same(with_bones, _expected(kp, ps, sk, 70., (64, 64), 0.64, bones_2d=True))


def test_device_downsample_is_the_reference_downsample():
    rng = np.random.default_rng(6)
    for factor in (2, 3, 8):
        x = (rng.standard_normal((41, 2, 17, 2)) * 300).astype(np.float32)
        got = R.downsample_frames(torch.from_numpy(x).cuda(), factor).cpu().numpy()
        assert np.array_equal(got.view(np.uint32), RR.downsample(x, factor).view(np.uint32))
        assert np.array_equal(got.view(np.uint32), RR.reference_downsample(x, factor).view(np.uint32))
        v = rng.integers(0, 256, (17, 9, 11, 3), dtype=np.uint8)
        got = R.downsample_frames(torch.from_numpy(v).cuda(), factor).cpu().numpy()
        assert np.array_equal(got, RR.reference_downsample(v, factor).astype('uint8'))


def _big_scene(rng, **kw):
    video = rng.integers(0, 256, (40, 72, 128, 3), dtype=np.uint8)
    kp = _keypoints(rng, 40, 2, 17, 128, 72)
    ps = {'a': _poses(rng, 40, 17, x0=-0.5), 'b': _poses(rng, 40, 17, x0=0.5)}
    return R.Scene(kp, ps, _Skel(H36M), 70., (128, 72), size=0.96, input_frames=video, keypoints_metadata=META, **kw)


def test_frame_ranges_and_repeated_calls_give_the_same_bytes():
    rng = np.random.default_rng(7)
    for kw in ({}, {'com_reconstrcution': True}, {'downsample': 3}):
        sc = _big_scene(rng, **kw)
        whole = sc.render()
        again = sc.render()
        assert torch.equal(whole, again)
        n = sc.n_frames
        parts = torch.cat([sc.render(range(a, min(a + 7, n))) for a in range(0, n, 7)])
        assert torch.equal(whole, parts)
        assert torch.equal(sc.render((n - 1, n))[0], whole[n - 1])
    with pytest.raises(GastError, match='contiguous range'):
        sc.render(range(0, n + 1))


def test_render_frames_makes_no_host_sync():
    rng = np.random.default_rng(8)
    video = rng.integers(0, 256, (12, 36, 64, 3), dtype=np.uint8)
    kp, ps = _keypoints(rng, 12, 1, 17, 64, 36), {'r': _poses(rng, 12, 17), 'g': _poses(rng, 12, 17)}
    dkp, dps = torch.from_numpy(kp).cuda(), {k: torch.from_numpy(v).cuda() for k, v in ps.items()}
    dvid = torch.from_numpy(video).cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        a = R.render_frames(kp, ps, _Skel(H36M), 70., (64, 36), size=0.64, input_frames=video, downsample=2,
                            input_video_skip=1, keypoints_metadata=META)
        b = R.render_frames(dkp, dps, _Skel(H36M), 70., (64, 36), size=0.64, input_frames=dvid, downsample=2,
                            input_video_skip=1, keypoints_metadata=META, frames=range(1, 4))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a[1:4], b)


def _stub_ffmpeg(tmp_path, monkeypatch):
    """an `ffmpeg` on PATH that copies its stdin to a file"""
    sink = tmp_path / 'piped.rgb'
    exe = tmp_path / 'bin' / 'ffmpeg'
    exe.parent.mkdir()
    exe.write_text('#!/bin/sh\ncat > "%s"\n' % sink)
    exe.chmod(exe.stat().st_mode | stat.S_IXUSR)
    monkeypatch.setenv('PATH', str(exe.parent) + os.pathsep + os.environ.get('PATH', ''))
    return sink


def test_render_animation_pipes_the_frames_to_ffmpeg(tmp_path, monkeypatch):
    from device.tools import vis_h36m, visualization
    rng = np.random.default_rng(9)
    kp = _keypoints(rng, 70, 2, 17, 96, 64)
    ps = {'Reconstruction 1': _poses(rng, 70, 17, x0=-0.6), 'Reconstruction 2': _poses(rng, 70, 17, x0=0.6)}
    sk = _Skel(H36M)
    sink = _stub_ffmpeg(tmp_path, monkeypatch)
    vis_h36m.render_animation(kp, META, ps, sk, 25, 30000, np.array(70., dtype=np.float32), str(tmp_path / 'o.mp4'),
                              (96, 64), size=0.64, com_reconstrcution=True)
    want = R.render_frames(kp, ps, sk, 70., (96, 64), size=0.64, com_reconstrcution=True, keypoints_metadata=META)
    assert sink.read_bytes() == want.cpu().numpy().tobytes()
    # trainval.py --render: visualization.py's (T, J, 2) keypoints, two panels following the root, downsampled
    gt = {'Reconstruction': _poses(rng, 70, 17, walk=0.05), 'Ground truth': _poses(rng, 70, 17, walk=0.05)}
    visualization.render_animation(kp[:, 0], META, gt, sk, 50, 3000, 30., str(tmp_path / 'o.mp4'), (96, 64),
                                   limit=-1, downsample=2, size=0.64)
    want = R.render_frames(kp[:, 0], gt, sk, 30., (96, 64), size=0.64, downsample=2, follow_root=True,
                           keypoints_metadata=META)
    assert sink.read_bytes() == want.cpu().numpy().tobytes()
    monkeypatch.setenv('PATH', str(tmp_path / 'nothing'))
    with pytest.raises(GastError, match='ffmpeg was not found on PATH'):
        vis_h36m.render_animation(kp, META, ps, sk, 25, 3000, 70., str(tmp_path / 'o.mp4'), (96, 64), size=0.64)
