"""numpy restatement of the dataset-preparation kernels' arithmetic (csrc/pipeline.cuh: world_to_camera_kernel,
project_to_2d_kernel, screen_norm_seg_kernel, kpt_convert_kernel mode 3), float32 operation by operation, and the
synthetic Human3.6M / HumanEva inputs of tests/golden/make_golden_dataset.py.  tests/test_dataset_cpu.py holds it to
the reference's goldens bit for bit."""
import os

import numpy as np

f32, f64 = np.float32, np.float64
H36M_REMOVED = [4, 5, 9, 10, 11, 16, 20, 21, 22, 23, 24, 28, 29, 30, 31]    # h36m_dataset.py, 'cpn_ft_h36m_dbb'
H36M_KEPT = [j for j in range(32) if j not in H36M_REMOVED]


def fma32(a, b, c):
    """float32 fma(a, b, c), correctly rounded: a*b is exact in double, the double sum's error is recovered exactly
    (TwoSum) and decides the rounding when the double sum sits on a float32 midpoint"""
    a, b, c = (np.asarray(v, f64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    r = s.astype(f32)
    rd = r.astype(f64)
    other = np.where(rd < s, np.nextafter(r, f32(np.inf)), np.nextafter(r, f32(-np.inf))).astype(f64)
    tie = (rd != s) & ((s - rd) == (other - s)) & (err != 0)
    return np.where(tie, np.where(err > 0, np.maximum(rd, other), np.minimum(rd, other)), rd).astype(f32)


def _cross(q, v):
    """torch's CPU cross(q, v) for one q (3,) and v (...,3): component i = fma(q[i+1], v[i+2], -(q[i+2] * v[i+1]))"""
    return np.stack([fma32(q[(i + 1) % 3], v[..., (i + 2) % 3], -(q[(i + 2) % 3] * v[..., (i + 1) % 3]))
                     for i in range(3)], -1)


def world_to_camera(X, R, t, root_relative=False):
    """camera.py:22-24 (+ main.py:33 with root_relative), X (..., J, 3) float32"""
    R, t = np.asarray(R, f32), np.asarray(t, f32)
    v = (np.asarray(X, f32) - t).astype(f32)
    q = -R[1:]
    u = _cross(q, v)
    w = _cross(q, u)
    out = (v + f32(2) * (R[0] * u + w)).astype(f32)
    if root_relative:
        out[..., 1:, :] -= out[..., :1, :]
    return out


def project_to_2d(X, cam):
    """camera.py:31-62: X (N, ..., 3), cam (N, 9)"""
    X = np.asarray(X, f32)
    k = np.asarray(cam, f32).reshape((cam.shape[0],) + (1,) * (X.ndim - 2) + (9,))
    xx, yy = X[..., 0] / X[..., 2], X[..., 1] / X[..., 2]
    r2 = xx * xx + yy * yy
    r4 = r2 * r2
    r6 = r4 * r2
    radial = f32(1) + ((k[..., 4] * r2 + k[..., 5] * r4) + k[..., 6] * r6)
    tan = k[..., 7] * xx + k[..., 8] * yy
    rt = radial + tan
    u = xx * rt + k[..., 7] * r2
    v = yy * rt + k[..., 8] * r2
    return np.stack([k[..., 0] * u + k[..., 2], k[..., 1] * v + k[..., 3]], -1).astype(f32)


def normalize_screen(X, w, h, from_image=False):
    """camera.py:8-12 on channels 0 and 1 of X (..., F>=2), the result rounded to float32 as main.py:101 stores it;
    from_image first takes the points through image_coordinates (:15-19) and float32"""
    X = np.array(X, f32)
    off = np.array([1, h / w], f64)
    xy = X[..., :2]
    if from_image:
        xy = ((xy.astype(f64) + off) * w / 2).astype(f32)
    X[..., :2] = ((xy / f32(w) * f32(2)).astype(f64) - off).astype(f32)
    return X


def coco_humaneva15(kps):
    """main.py:80-95 (float32 (T, 17, F) -> (T, 15, F))"""
    k15 = np.zeros((kps.shape[0], 15, kps.shape[2]), f32)
    k15[:, 0] = (kps[:, 11] + kps[:, 12]) / f32(2)
    k15[:, 1] = (kps[:, 5] + kps[:, 6]) / f32(2)
    k15[:, 2:] = kps[:, [5, 7, 9, 6, 8, 10, 11, 13, 15, 12, 14, 16, 0]]
    return k15


# ------------------------------------------------------------------------------------------------------------------
# synthetic inputs: positions_3d and positions_2d dicts as the npz files hold them (metres / pixels, float32)
# ------------------------------------------------------------------------------------------------------------------
def _motion(rs, T, J):
    root = np.cumsum(rs.standard_normal((T, 1, 3)) * 0.01, 0) + rs.uniform(-1, 1, (1, 1, 3)) * [1, 1, 0] + [0, 0, 0.9]
    return (root + rs.standard_normal((1, J, 3)) * 0.4 + rs.standard_normal((T, J, 3)) * 0.02).astype(f32)


def synth_h36m(seed=3):
    rs = np.random.RandomState(seed)
    acts = {'S1': [('Walking', 41), ('Walking 1', 37), ('Eating 2', 23)], 'S9': [('Directions', 30), ('Walking', 19)]}
    pos3d, pos2d = {}, {}
    for s, al in acts.items():
        pos3d[s], pos2d[s] = {}, {}
        for a, T in al:
            pos3d[s][a] = _motion(rs, T, 32)
            pos2d[s][a] = [rs.uniform(0, 1000, (T + int(rs.randint(0, 6)), 17, 2)).astype(f32) for _ in range(4)]
    return pos3d, pos2d


def synth_humaneva(seed=4):
    rs = np.random.RandomState(seed)
    acts = {'Train/S1': [('Walking 1 chunk0', 29), ('Jog 1 chunk0', 21)], 'Validate/S2': [('Walking 1 chunk1', 26)]}
    pos3d, pos2d = {}, {}
    for s, al in acts.items():
        pos3d[s], pos2d[s] = {}, {}
        for a, T in al:
            pos3d[s][a] = _motion(rs, T, 15)
            pos2d[s][a] = [rs.uniform(0, 640, (T + int(rs.randint(0, 6)), 17, 2)).astype(f32) for _ in range(3)]
    return pos3d, pos2d


def write_data(root, name, keypoints_type, pos3d, pos2d):
    """root/data/data_3d_<name>.npz and data_2d_<name>_<keypoints_type>.npz as main.load_data reads them"""
    os.makedirs(os.path.join(root, 'data'), exist_ok=True)
    np.savez_compressed(os.path.join(root, 'data', 'data_3d_%s.npz' % name), positions_3d=pos3d)
    np.savez_compressed(os.path.join(root, 'data', 'data_2d_%s_%s.npz' % (name, keypoints_type)), positions_2d=pos2d,
                        metadata={'layout_name': 'coco', 'num_joints': 17,
                                  'keypoints_symmetry': [[1, 3, 5, 7, 9, 11, 13, 15], [2, 4, 6, 8, 10, 12, 14, 16]]})


def split(g, key):
    """a golden's flattened list back into its arrays"""
    return np.split(g[key], np.cumsum(g[key + '_len'])[:-1]) if key in g else None


class MocapStandIn(object):
    """what gast_b200.dataset.prepare reads of a MocapDataset: subjects(), [subject][action] = {'positions', 'cameras'},
    cameras()"""

    def __init__(self, positions, cameras):
        self._cameras = cameras
        self._data = {s: {a: {'positions': p, 'cameras': cameras[s]} for a, p in acts.items()}
                      for s, acts in positions.items()}

    def __getitem__(self, key):
        return self._data[key]

    def subjects(self):
        return self._data.keys()

    def cameras(self):
        return self._cameras
