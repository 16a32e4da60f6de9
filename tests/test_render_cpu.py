"""CPU checks of the animation renderer (gast_b200.render, csrc/render.cuh; DESIGN.md §8.5):
  * the bone colour table is h36m_color_edge's with the RGB values its comments give;
  * gast_render_geometry is DESIGN.md §8.5's view, image fit and coverage formulas, and projects the axis box inside
    the panel with its centre at the panel's centre and z up;
  * the numpy restatement's downsample equals the reference's downsample_tensor expression bit for bit;
  * the argument refusals of render_frames, gast_render_frames and render_animation, all before any launch."""
import ctypes as C
import os
import sys
import types

import numpy as np
import pytest

import renderref as RR
from conftest import REPO
from gast_b200 import _lib as L
from gast_b200 import render as R
from gast_b200.engine import GastError

# matplotlib's named colours that h36m_color_edge returns, as the comments of tools/color_edge.py give them
CSS = {'peru': (205, 133, 63), 'indianred': (205, 92, 92), 'coral': (255, 127, 80), 'brown': (165, 42, 42),
       'tan': (210, 180, 140), 'olive': (128, 128, 0), 'purple': (128, 0, 128)}
H36M_EDGE = {5: 'peru', 15: 'peru', 2: 'indianred', 12: 'indianred', 6: 'coral', 16: 'coral', 3: 'brown',
             13: 'brown', 1: 'tan', 4: 'tan', 11: 'tan', 14: 'tan', 7: 'olive', 9: 'olive'}
REF = os.path.join(REPO, 'oracle', '_ref')


def test_color_table_is_h36m_color_edge():
    t = R.color_table(32)
    for j in range(32):
        assert tuple(t[j]) == CSS[H36M_EDGE.get(j, 'purple')], j


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, 'tools', 'visualization.py')),
                    reason='reference caller files not staged')
def test_color_table_is_the_reference_color_edge(monkeypatch):
    """tools/visualization.py's color_edge groups the joints as h36m_color_edge does"""
    for name in ('matplotlib', 'matplotlib.pyplot', 'matplotlib.animation', 'mpl_toolkits', 'mpl_toolkits.mplot3d'):
        monkeypatch.setitem(sys.modules, name, sys.modules.get(name) or types.ModuleType(name))
    monkeypatch.setattr(sys.modules['matplotlib'], 'use', lambda *a, **k: None, raising=False)
    monkeypatch.setattr(sys.modules['matplotlib.animation'], 'FuncAnimation', object, raising=False)
    monkeypatch.setattr(sys.modules['matplotlib.animation'], 'writers', {}, raising=False)
    monkeypatch.setattr(sys.modules['mpl_toolkits.mplot3d'], 'Axes3D', object, raising=False)
    import importlib.util
    spec = importlib.util.spec_from_file_location('_ref_visualization', os.path.join(REF, 'tools', 'visualization.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    t = R.color_table(32)
    for j in range(32):
        assert tuple(t[j]) == CSS[mod.color_edge(j)], j


def _design_view(S, azim, shared, elev=15., radius=1.7, dist=7.5):
    """DESIGN.md §8.5 in float64: (rows (3,4), box lo, box hi)"""
    a, e = np.radians(azim), np.radians(elev)
    r = np.array([-np.sin(a), np.cos(a), 0.])
    u = np.array([-np.sin(e) * np.cos(a), -np.sin(e) * np.sin(a), np.cos(e)])
    w = np.array([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)])
    xy = radius if shared else radius / 2
    lo, hi = np.array([-xy, -xy, 0.]), np.array([xy, xy, radius])
    span, c = hi - lo, (hi + lo) / 2
    h = np.sqrt(3) / 2
    k = S / 2 * (dist - h) / (h * dist)
    rows = np.zeros((3, 4))
    rows[0, :3], rows[1, :3], rows[2, :3] = k * r / span, -k * u / span, -w / (dist * span)
    rows[:, 3] = -rows[:, :3] @ c
    rows[2, 3] += 1
    return rows, lo, hi


@pytest.mark.parametrize('azim', [70., -90., 0., 135.5])
@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('S', [64, 500])
def test_geometry_is_the_design_view(azim, shared, S):
    geo = R.geometry(S, 100, 480, 640, azim, shared)
    rows, lo, hi = _design_view(S, azim, shared)
    np.testing.assert_allclose(geo[:12].reshape(3, 4), rows, rtol=1e-6, atol=1e-5 * S)
    assert geo[19] == S / 2
    corners = np.array([[x, y, z, 1.] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
    p = corners @ rows.T
    X, Y = S / 2 + p[:, 0] / p[:, 2], S / 2 + p[:, 1] / p[:, 2]
    assert np.all(p[:, 2] > 0)
    assert np.all(np.hypot(X - S / 2, Y - S / 2) <= S / 2 + 1e-9)          # the box's bounding sphere fits
    centre = np.append((lo + hi) / 2, 1.) @ rows.T
    assert abs(centre[0] / centre[2]) < 1e-9 and abs(centre[1] / centre[2]) < 1e-9
    top = np.array([0., 0., hi[2], 1.]) @ rows.T
    bottom = np.array([0., 0., lo[2], 1.]) @ rows.T
    assert top[1] / top[2] < bottom[1] / bottom[2]                       # z is up on the screen
    # the restatement's float32 projection of the corners agrees with the float64 formula
    q = RR._project(corners[:, :3].astype(np.float32), geo, False)
    np.testing.assert_allclose(q[:, 0], X, atol=1e-3)
    np.testing.assert_allclose(q[:, 1], Y, atol=1e-3)


def test_geometry_image_fit_and_coverage():
    for (H, W), (scale, ox, oy) in {(1080, 1920): (500 / 1920, 0., 500 * 840 / 3840),
                                    (1920, 1080): (500 / 1920, 500 * 840 / 3840, 0.),
                                    (500, 500): (1., 0., 0.)}.items():
        geo = R.geometry(500, 100, H, W, 70.)
        assert geo[12] == np.float32(scale) and geo[13] == np.float32(ox) and geo[14] == np.float32(oy)
    geo = R.geometry(500, 100, 1000, 1000, 70.)
    px = 100 / 72
    rd, ew = np.sqrt(10) / 2 * px, 1.5 * px
    assert geo[15] == np.float32(3 * px / 2 + .5) and geo[16] == np.float32(1.5 * px / 2 + .5)
    assert geo[17] == np.float32(rd - ew / 2 + .5) and geo[18] == np.float32(rd + ew / 2 + .5)


@pytest.mark.parametrize('factor', [2, 3, 5, 8, 9, 16])    # the reference downsamples when factor > 1
def test_downsample_restatement_is_the_reference_expression(factor):
    rng = np.random.default_rng(factor)
    for shape in [(37, 2, 17, 2), (50, 17, 3), (29, 19, 3)]:
        x = (rng.standard_normal(shape) * 100).astype(np.float32)
        x[3] = -0.0
        ref = RR.reference_downsample(x, factor)
        got = RR.downsample(x, factor)
        assert ref.dtype == got.dtype == np.float32
        assert np.array_equal(ref.view(np.uint32), got.view(np.uint32))
    v = rng.integers(0, 256, (23, 5, 7, 3), dtype=np.uint8)
    assert np.array_equal(RR.reference_downsample(v, factor).astype('uint8'), RR.downsample(v, factor))


class _Skel(object):
    def __init__(self, parents):
        self._p = parents

    def parents(self):
        return np.array(self._p)

    def joints_right(self):
        return [1, 2, 3, 14, 15, 16]


H36M = [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15]


def _args(T=6, M=1, J=17):
    return np.zeros((T, M, J, 2), np.float32), {'Reconstruction': np.zeros((T, J, 3), np.float32)}


def test_render_frames_refusals():
    import torch
    kp, poses = _args()
    sk = _Skel(H36M)
    for kw, what in [(dict(keypoints=np.zeros((6, 17, 3))), 'keypoints'),
                     (dict(poses={}), 'at least one'),
                     (dict(poses={'a': np.zeros((6, 16, 3))}), 'poses'),
                     (dict(skeleton=_Skel(H36M[:16])), 'skeleton has'),
                     (dict(skeleton=_Skel([-1] + [20] * 16)), 'parents'),
                     (dict(keypoints=np.zeros((6, 16, 17, 2))), 'persons'),
                     (dict(keypoints=torch.zeros(6, 17, 2)), 'no CPU path'),
                     (dict(downsample=0), 'downsample'),
                     (dict(input_video_skip=-1), 'input_video_skip'),
                     (dict(viewport=(0, 10)), 'input image'),
                     (dict(size=0.01), 'pixels'),
                     (dict(input_frames=np.zeros((6, 10, 10))), 'input_frames'),
                     (dict(poses={str(i): np.zeros((6, 17, 3)) for i in range(9)}), 'panels'),
                     (dict(keypoints_metadata={'keypoints_symmetry': ([], [17]), 'layout_name': 'h36m'}), 'right')]:
        a = dict(keypoints=kp, poses=poses, skeleton=sk, azim=70., viewport=(64, 48))
        a.update(kw)
        with pytest.raises(GastError, match=what):
            R.render_frames(a.pop('keypoints'), a.pop('poses'), a.pop('skeleton'), a.pop('azim'), a.pop('viewport'), **a)
    with pytest.raises(GastError, match='shared panel'):
        R.render_frames(np.zeros((6, 2, 17, 2)), poses, sk, 70., (64, 48), com_reconstrcution=True, follow_root=True)


def test_gast_render_frames_refusals():
    lib = L.load()
    J = 17
    par = (C.c_int32 * 32)(*(H36M + [0] * 15))
    col = (C.c_uint8 * 96)()
    right = (C.c_int32 * 2)(1, 2)
    fake = C.c_void_p(256)

    def call(**kw):
        a = dict(kp=fake, n_kp=10, M=1, J=J, poses=fake, n_pose=1, n_pose_frames=10, video=None, n_video=0, H=48, W=64,
                 par=par, col=col, right=right, n_right=2, n_bones=17, S=64, dpi=100., flags=0, f0=0, F=10, out=fake)
        a.update(kw)
        return lib.gast_render_frames(a['kp'], a['n_kp'], a['M'], a['J'], a['poses'], a['n_pose'], a['n_pose_frames'],
                                      a['video'], a['n_video'], a['H'], a['W'], a['par'], a['col'], a['right'],
                                      a['n_right'], a['n_bones'], a['S'], a['dpi'], 15., 70., 1.7, 7.5, a['flags'],
                                      a['f0'], a['F'], a['out'], None)

    for kw, what in [(dict(J=33), 'bad arguments'), (dict(n_bones=18), 'bad arguments'), (dict(F=0), 'bad arguments'),
                     (dict(flags=8), 'bad arguments'), (dict(M=16), 'exceed'), (dict(n_pose=9), '3D panels'),
                     (dict(flags=3), 'shared panel'), (dict(F=11), 'exceed the inputs'),
                     (dict(f0=5, F=6, n_pose_frames=20), 'exceed the inputs'),
                     (dict(video=fake, n_video=9), 'exceed the inputs'),
                     (dict(par=(C.c_int32 * 32)(*([-1] + [17] * 31))), 'parents'),
                     (dict(right=(C.c_int32 * 2)(1, 17)), 'right joint'), (dict(S=4), 'S <= 8192'),
                     (dict(dpi=0.), 'dpi')]:
        assert call(**kw) != 0, kw
        assert what in L.last_error(), (kw, L.last_error())
    assert lib.gast_downsample_frames(fake, 10, 6, 0, 0, fake, None) != 0
    assert lib.gast_downsample_frames(fake, 10, 6, 2, 2, fake, None) != 0


def test_render_animation_refusals(tmp_path, monkeypatch):
    from device.tools import vis_h36m, visualization
    kp, poses = _args()
    meta = {'keypoints_symmetry': ([4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]), 'layout_name': 'h36m'}
    sk = _Skel(H36M)
    with pytest.raises(GastError, match='gif'):
        vis_h36m.render_animation(kp, meta, poses, sk, 25, 3000, 70., str(tmp_path / 'a.gif'), (64, 48))
    with pytest.raises(ValueError, match='Unsupported output format'):
        visualization.render_animation(kp[:, 0], meta, poses, sk, 25, 3000, 70., str(tmp_path / 'a.avi'), (64, 48))
    monkeypatch.setenv('PATH', str(tmp_path))
    for mod, k in ((vis_h36m, kp), (visualization, kp[:, 0])):
        with pytest.raises(GastError, match='ffmpeg was not found on PATH'):
            mod.render_animation(k, meta, poses, sk, 25, 3000, 70., str(tmp_path / 'a.mp4'), (64, 48))
