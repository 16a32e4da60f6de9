"""Mocap datasets prepared on the device: what trainval.py gets from `main.load_data` and `main.fetch` (main.py:12-159),
and the `-k gt` keypoints of data/prepare_data_h36m.py:113-121, as CUDA tensors.

`prepare(dataset, keypoints)` takes the caller's loaded `Human36mDataset` / `HumanEvaDataset` and its `positions_2d`
dict, checks on the host what main.py's asserts check, uploads every mocap sequence once and every detection array
once, and then launches:

- one `gast_world_to_camera` for every (sequence, camera): camera-space poses, root-relative (main.py:29-35);
- one `gast_normalize_screen_segments` for every detection array: trimmed to the mocap length and normalised with its
  own camera's resolution (main.py:59-102), after one `gast_keypoints_convert` for HumanEva's COCO -> 15 joints.

The results equal main.load_data's bit for bit for float32 input.  Nothing is read back: the returned
`PreparedDataset` holds views into three device buffers, and `fetch`, `test_set` and `ground_truth_2d` hand out views
(or launch) without a host synchronisation, ready for `device.common.generators`, `training.EpochTrainer` and
`evaluation.evaluate_sequences`.  The caller's objects are not modified.
"""
import numpy as np
import torch

from . import pipeline as _P
from .engine import GastError


def _f32(a, shape_ok, what):
    if not isinstance(a, np.ndarray) or a.dtype != np.float32 or not shape_ok(a.shape):
        raise GastError('prepare: %s must be a float32 numpy array, got %s' % (
            what, (a.dtype, a.shape) if isinstance(a, np.ndarray) else type(a).__name__))
    return a


def _upload(arrays, shape, dtype, dev):
    """the arrays concatenated along axis 0 into one new device tensor (n, *shape): one copy per array, no host wait"""
    out = torch.empty((sum(int(a.shape[0]) for a in arrays),) + tuple(shape), dtype=dtype, device=dev)
    o = 0
    for a in arrays:
        n = int(a.shape[0])
        if n:
            out[o:o + n].copy_(torch.from_numpy(np.ascontiguousarray(a)).reshape((n,) + tuple(shape)), non_blocking=True)
        o += n
    return out


def _offsets(lengths):
    return np.concatenate([[0], np.cumsum(lengths, dtype=np.int64)]).astype(np.int64)


class PreparedDataset(object):
    """A dataset after main.load_data, on the device.

    positions_3d[subject][action]: per camera a CUDA (T, J, 3) camera-space pose sequence, joints 1.. relative to
    joint 0 (only actions with mocap positions); keypoints[subject][action]: per camera the CUDA (T, J2, F) normalised
    keypoints, trimmed to the mocap length; intrinsics[subject]: per camera its CUDA (9,) intrinsics, or None."""

    def __init__(self, positions_3d, keypoints, intrinsics, actions, gt=None):
        self.positions_3d = positions_3d
        self.keypoints = keypoints
        self.intrinsics = intrinsics
        self._actions = actions           # dataset[subject].keys() in order
        self._gt = gt                     # what ground_truth_2d launches from

    def ground_truth_2d(self):
        """The same dataset with the ground-truth keypoints in place of the detections: what `-k gt` loads
        (prepare_data_h36m.py:113-121 world_to_camera -> project_to_2d -> image_coordinates -> float32, then main.py:101
        normalize_screen_coordinates), for every (subject, action, camera) with mocap positions, in the dataset's
        order.  Three launches; the cameras need intrinsics."""
        g = self._gt
        if g is None or g['n'] == 0:
            raise GastError('ground_truth_2d: the dataset has no mocap positions')
        if g['intr'] is None:
            raise GastError('ground_truth_2d: every camera with mocap positions needs intrinsics (a HumanEva camera has '
                            'none)')
        src, dst = g['src'], g['dst']
        cam = _P.world_to_camera_segments(g['x'], src, dst, g['qt'], g['n'])
        px = _P.project_to_2d_segments(cam.reshape(-1, 3), dst * cam.shape[1], g['intr'])
        kp = _P.normalize_screen_segments(px.reshape(cam.shape[0], cam.shape[1], 2), dst[:-1], dst, g['wh'], g['n'],
                                          from_image=True)
        keypoints = {}
        for (subject, action, T, ncam), o in zip(g['seqs'], g['seq_dst']):
            keypoints.setdefault(subject, {})[action] = [kp[o + c * T:o + (c + 1) * T] for c in range(ncam)]
        return PreparedDataset(self.positions_3d, keypoints, self.intrinsics, self._actions, g)

    def _check_subject(self, subject, what):
        if subject not in self.keypoints:
            raise GastError('%s: subject %s is not in the keypoints' % (what, subject))

    def fetch(self, subjects, action_filter=None, downsample=5, subset=1, parse_3d_poses=True):
        """main.fetch (main.py:107-159): (camera intrinsics, 3D poses, 2D keypoints) lists of CUDA views in its order,
        None where it returns None; downsampled views are strided.  subset < 1 is refused: the reference's
        deterministic_random raises there (tools/utils.py:56)."""
        if subset < 1:
            raise GastError('fetch: subset < 1 is not supported (the reference raises in deterministic_random)')
        out_poses_3d, out_poses_2d, out_camera_params = [], [], []
        for subject in subjects:
            self._check_subject(subject, 'fetch')
            for action in self.keypoints[subject].keys():
                if action_filter is not None and not any(action.startswith(a) for a in action_filter):
                    continue
                poses_2d = self.keypoints[subject][action]
                out_poses_2d.extend(poses_2d)
                if subject in self.intrinsics:
                    cams = self.intrinsics[subject]
                    if len(cams) != len(poses_2d):
                        raise GastError('fetch: Camera count mismatch (%s %s)' % (subject, action))
                    out_camera_params.extend(c for c in cams if c is not None)
                if parse_3d_poses:
                    if action not in self._actions.get(subject, ()):
                        raise GastError('fetch: action %s of subject %s is not in the dataset' % (action, subject))
                    poses_3d = self.positions_3d.get(subject, {}).get(action)
                    if poses_3d is not None:
                        if len(poses_3d) != len(poses_2d):
                            raise GastError('fetch: Camera count mismatch (%s %s)' % (subject, action))
                        out_poses_3d.extend(poses_3d)
        stride = int(downsample)
        if stride > 1:
            out_poses_2d = [p[::stride] for p in out_poses_2d]
            out_poses_3d = [p[::stride] for p in out_poses_3d]
        return (out_camera_params or None), (out_poses_3d or None), out_poses_2d

    def test_set(self, subjects, action_filter=None, by_subject=False, downsample=1):
        """The sequences trainval.py's evaluation scores (trainval.py:263-337): (poses_3d, poses_2d, groups), one entry
        per (subject, action, camera) in run_evaluation's order, grouped by action name (`action.split(' ')[0]`), or
        by (subject, action name) with by_subject.  Pass them to evaluation.evaluate_sequences(..., groups=groups)."""
        groups = {}
        for subject in subjects:
            self._check_subject(subject, 'test_set')
            for action in self._actions.get(subject, ()):
                name = action.split(' ')[0]
                groups.setdefault((subject, name) if by_subject else name, []).append((subject, action))
        poses_3d, poses_2d, labels = [], [], []
        stride = int(downsample)
        for key in groups:
            name = key[1] if by_subject else key
            if action_filter is not None and not any(name.startswith(a) for a in action_filter):
                continue
            for subject, action in groups[key]:
                p2 = self.keypoints[subject][action]
                p3 = self.positions_3d.get(subject, {}).get(action)
                if p3 is None or len(p3) != len(p2):
                    raise GastError('test_set: %s %s needs one 3D sequence per camera' % (subject, action))
                poses_2d.extend(p[::stride] if stride > 1 else p for p in p2)
                poses_3d.extend(p[::stride] if stride > 1 else p for p in p3)
                labels.extend([key] * len(p2))
        return poses_3d, poses_2d, labels


def prepare(dataset, keypoints, humaneva=False, device='cuda'):
    """main.load_data's preparation (main.py:24-104) of `dataset` (a loaded Human36mDataset or HumanEvaDataset) and
    `keypoints` (its positions_2d dict) on `device`: returns a PreparedDataset.  humaneva=True remaps the 17 COCO
    detections to HumanEva's 15 joints first (main.py:79-98).  Positions and detections must be float32 (as the
    reference's npz files hold them); HumanEva detections (T, 17, 2).  Everything main.py asserts, and every lookup its
    loops would fail, is checked before the first upload."""
    dev = torch.device(device)
    cams = dataset.cameras()
    actions = {s: list(dataset[s].keys()) for s in dataset.subjects()}
    # 3D: every (subject, action) with mocap positions, every camera of it (main.py:25-35, 51-68)
    seqs, pos, qt, intr, wh3, mocap = [], [], [], [], [], {}
    for subject in dataset.subjects():
        if subject not in keypoints:
            raise GastError('prepare: subject %s is missing from the 2D detections dataset' % subject)
        for action in actions[subject]:
            if action not in keypoints[subject]:
                raise GastError('prepare: action %s of subject %s is missing from the 2D detections dataset'
                                % (action, subject))
            anim = dataset[subject][action]
            if 'positions' not in anim:
                continue
            p = _f32(anim['positions'], lambda s: len(s) == 3 and s[2] == 3, 'positions of %s %s' % (subject, action))
            T, ncam = int(p.shape[0]), len(anim['cameras'])
            kp = keypoints[subject][action]
            if len(kp) != ncam:
                raise GastError('prepare: %s %s has %d detection cameras and %d mocap cameras' % (subject, action,
                                                                                               len(kp), ncam))
            for c, cam in enumerate(anim['cameras']):
                if 'orientation' not in cam or 'translation' not in cam:
                    raise GastError('prepare: camera %d of %s has no extrinsics' % (c, subject))
                if kp[c].shape[0] < T:
                    raise GastError('prepare: %s %s camera %d has %d detected frames for %d mocap frames'
                                    % (subject, action, c, kp[c].shape[0], T))
                qt.append(np.concatenate([np.asarray(cam['orientation'], np.float32).reshape(4),
                                          np.asarray(cam['translation'], np.float32).reshape(3)]))
                intr.append(np.asarray(cam['intrinsic'], np.float32).reshape(9) if 'intrinsic' in cam else None)
                wh3.append((cam['res_w'], cam['res_h'] / cam['res_w']))
            seqs.append((subject, action, T, ncam))
            pos.append(p)
            mocap[(subject, action)] = T
    if len({int(p.shape[1]) for p in pos}) > 1:
        raise GastError('prepare: the mocap sequences have different joint counts')
    # 2D: every detection array (main.py:70-102), trimmed to its mocap length
    raw, seg2, shape2 = [], [], None
    for subject in keypoints:
        if subject not in cams:
            raise GastError('prepare: subject %s of the detections has no cameras' % subject)
        for action in keypoints[subject]:
            for c, kps in enumerate(keypoints[subject][action]):
                if c >= len(cams[subject]):
                    raise GastError('prepare: %s %s has detections for camera %d, which subject %s lacks'
                                    % (subject, action, c, subject))
                _f32(kps, lambda s: len(s) == 3 and s[2] >= 2, 'detections of %s %s' % (subject, action))
                if humaneva and kps.shape[1:] != (17, 2):
                    raise GastError('prepare: HumanEva detections must be (T, 17, 2), got %s' % (kps.shape,))
                if shape2 is not None and kps.shape[1:] != shape2:
                    raise GastError('prepare: detections of different shapes %s and %s' % (shape2, kps.shape[1:]))
                shape2 = kps.shape[1:]
                cam = cams[subject][c]
                seg2.append((subject, action, c, mocap.get((subject, action), int(kps.shape[0])),
                             (cam['res_w'], cam['res_h'] / cam['res_w'])))
                raw.append(kps)
    intr_tab = {}
    for subject, cl in cams.items():
        intr_tab[subject] = [np.asarray(c['intrinsic'], np.float32).reshape(9) if 'intrinsic' in c else None for c in cl]

    # uploads: the data once, the tables in three tensors
    S3, S2 = len(qt), len(seg2)
    src3 = np.repeat(_offsets([s[2] for s in seqs])[:-1], [s[3] for s in seqs])
    dst3 = _offsets([s[2] for s in seqs for _ in range(s[3])])
    src2 = _offsets([int(k.shape[0]) for k in raw])[:-1]
    dst2 = _offsets([s[3] for s in seg2])
    ints = _upload([np.concatenate([src3, dst3, src2, dst2]).astype(np.int64)], (), torch.int64, dev)
    src3_d, dst3_d = ints[:S3], ints[S3:2 * S3 + 1]
    src2_d, dst2_d = ints[2 * S3 + 1:2 * S3 + 1 + S2], ints[2 * S3 + 1 + S2:]
    have_intr = S3 > 0 and all(k is not None for k in intr)
    subj_intr = [k for cl in intr_tab.values() for k in cl if k is not None]
    floats = _upload([np.concatenate([np.asarray(qt, np.float32).reshape(-1),
                                      np.asarray(intr if have_intr else [], np.float32).reshape(-1),
                                      np.asarray(subj_intr, np.float32).reshape(-1)])], (), torch.float32, dev)
    qt_d = floats[:7 * S3].view(S3, 7)
    intr3_d = floats[7 * S3:16 * S3].view(S3, 9) if have_intr else None
    subj_d = floats[(16 if have_intr else 7) * S3:].view(-1, 9)
    doubles = _upload([np.asarray([s[4] for s in seg2] + wh3, np.float64).reshape(-1, 2)], (2,), torch.float64, dev)
    wh2_d, wh3_d = doubles[:S2], doubles[S2:]
    x3 = _upload(pos, pos[0].shape[1:], torch.float32, dev) if pos else None
    x2 = _upload(raw, shape2, torch.float32, dev) if raw else None

    # launches
    positions_3d = {}
    n3 = int(dst3[-1])
    if n3 > 0:
        p3 = _P.world_to_camera_segments(x3, src3_d, dst3_d, qt_d, n3, root_relative=True)
    seq_dst, o = [], 0
    for subject, action, T, ncam in seqs:
        seq_dst.append(o)
        if n3 > 0:
            positions_3d.setdefault(subject, {})[action] = [p3[o + c * T:o + (c + 1) * T] for c in range(ncam)]
        o += T * ncam
    kp_out = {}
    n2 = int(dst2[-1])
    if n2 > 0:
        src = _P.keypoints_convert(x2, _P.KPT_COCO_HUMANEVA)[0] if humaneva else x2
        k2 = _P.normalize_screen_segments(src, src2_d, dst2_d, wh2_d, n2)
    elif raw:
        k2 = torch.empty(((0, 15, 2) if humaneva else (0,) + tuple(shape2)), dtype=torch.float32, device=dev)
    for (subject, action, c, T, _), o in zip(seg2, dst2[:-1]):
        kp_out.setdefault(subject, {}).setdefault(action, []).append(k2[int(o):int(o) + T])
    for subject in keypoints:                      # actions and subjects without detections keep their (empty) entry
        for action in keypoints[subject]:
            kp_out.setdefault(subject, {}).setdefault(action, [])
    intrinsics, q = {}, 0
    for subject, cl in intr_tab.items():
        row = []
        for k in cl:
            row.append(subj_d[q] if k is not None else None)
            q += k is not None
        intrinsics[subject] = row
    gt = {'x': x3, 'src': src3_d, 'dst': dst3_d, 'qt': qt_d, 'n': n3, 'intr': intr3_d, 'wh': wh3_d, 'seqs': seqs,
          'seq_dst': seq_dst}
    return PreparedDataset(positions_3d, kp_out, intrinsics, actions, gt)
