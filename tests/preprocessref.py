"""numpy restatement of the video demo's keypoint repair and person placement (tools/preprocess.py:47-172), the
oracle of csrc/pipeline.cuh's h36m_coco_format, revise_kpts, revise_skes and revise_skes_real_time kernels.

TEST INFRASTRUCTURE ONLY.  Pinned bit for bit against the unmodified reference's outputs in
tests/golden/preprocess_17.npz (tests/golden/make_golden_preprocess.py) by tests/test_preprocess_cpu.py.
"""
import numpy as np

from oracle.pipeline_oracle import F32, _COCO_TO_H36M, coco_h36m

_LIMB = [1, 4, 11, 14]                               # the joints whose mean places a person


def _limb_mean(a):
    """mean over joints [1, 4, 11, 14] (axis -2) of (..., J, C): float32, left to right, then / 4"""
    s = a[..., 1, :].copy()
    for j in _LIMB[1:]:
        s = s + a[..., j, :]
    return s / F32(4)


def h36m_coco_format(keypoints, scores):
    """preprocess.py:47-75: the person slots with some non-zero coordinate -> (H36M keypoints (K,T,17,2),
    H36M scores (K,T,17), valid frame index arrays)."""
    kk, ss, frames = [], [], []
    for kp, sc in zip(np.asarray(keypoints, F32), np.asarray(scores, F32)):
        if not np.any(kp != 0):
            continue
        h, v = coco_h36m(kp)
        n = np.zeros_like(sc)
        for hj, cj in _COCO_TO_H36M.items():
            n[:, hj] = sc[:, cj]
        n[:, 0] = (sc[:, 11] + sc[:, 12]) / F32(2)
        n[:, 8] = (sc[:, 5] + sc[:, 6]) / F32(2)
        n[:, 7] = (n[:, 0] + n[:, 8]) / F32(2)
        n[:, 10] = (((sc[:, 1] + sc[:, 2]) + sc[:, 3]) + sc[:, 4]) / F32(4)
        kk.append(h)
        ss.append(n)
        frames.append(v)
    return np.asarray(kk, F32), np.asarray(ss, F32), frames


# low joints among [2, 3, 5, 6] -> (targets, sources) of the repair (preprocess.py:96-107)
_REPAIR = {(2, 3, 5, 6): ([2, 3, 5, 6], [1, 1, 4, 4]), (2, 3, 6): ([2, 3, 6], [1, 1, 5]), (3, 5, 6): ([3, 5, 6], [2, 4, 4]),
           (3, 6): ([3, 6], [2, 5]), (3,): ([3], [2]), (6,): ([6], [5])}


def revise_kpts(kpts, scores, valid_frames):
    """preprocess.py:78-112: zero outside the valid frames, the low-confidence (score < float32(0.3)) limb joints
    replaced at them by the first matching rule; every other combination leaves the pose unchanged."""
    kpts, scores = np.asarray(kpts, F32), np.asarray(scores, F32)
    out = np.zeros_like(kpts)
    for p, frames in enumerate(valid_frames):
        f = np.asarray(frames, np.int64).reshape(-1)
        k, s = kpts[p, f], scores[p, f]
        new = k.copy()
        low = s[:, [2, 3, 5, 6]] < F32(0.3)
        for key, (dst, src) in _REPAIR.items():
            rows = np.all(low == np.isin([2, 3, 5, 6], key), axis=1)
            new[np.ix_(rows, dst)] = k[rows][:, src]
        out[p, f] = new
    return out


def revise_skes(prediction, re_kpts, valid_frames):
    """preprocess.py:123-155: scatter, per-person 2D displacement / 500, the two-person split, z -= min z over the
    whole output (zero rows included).  ValueError when two persons share no valid frame."""
    re_kpts = np.asarray(re_kpts, F32)
    P, T, J = re_kpts.shape[:3]
    out = np.zeros((P, T, J, 3), F32)
    frames = [np.asarray(f, np.int64).reshape(-1) for f in valid_frames]
    for p, f in enumerate(frames):
        out[p, f] = np.asarray(prediction[p], F32)
        if f.size > 1:
            d = _limb_mean(re_kpts[p, f[1:], :, :2] - re_kpts[p, f[:1], :, :2])
            out[p, f[1:], :, 0] -= (d[:, 0] / F32(500))[:, None]
            out[p, f[1:], :, 1] += (d[:, 1] / F32(500))[:, None]
    if P == 2:
        common = frames[0][np.isin(frames[0], frames[1])]
        if not common.size:
            if frames[0].size or frames[1].size:
                raise ValueError('revise_skes: the two persons share no valid frame')
        else:
            t = common[0]
            a = _limb_mean(re_kpts[0, t, :, :2] - re_kpts[1, t, :, :2]) / F32(2)
            ax, ay = a[0] / F32(500), a[1] / F32(500)
            out[0, frames[0], :, 0] -= ax
            out[0, frames[0], :, 1] += ay
            out[1, frames[1], :, 0] += ax
            out[1, frames[1], :, 1] -= ay
    out[..., 2] -= out[..., 2].min()
    return out


def revise_skes_real_time(prediction, re_kpts, width):
    """preprocess.py:158-172: each person moved by its limb-mean image position, z -= min z over all persons."""
    pred = np.asarray(prediction, F32)
    if pred.shape[1:] != (17, 3):
        raise ValueError('revise_skes_real_time: (M,17,3) poses expected, got %s' % (pred.shape,))
    m = _limb_mean(np.asarray(re_kpts, F32)[:, :, :2])
    r = F32(500. * (width / 1920))
    out = pred.copy()
    out[:, :, 0] -= ((m[:, 0] - F32(3 * width / 5)) / r)[:, None]
    out[:, :, 1] += ((m[:, 1] - F32(width / 5)) / r)[:, None]
    out[:, :, 2] -= out[:, :, 2].min()
    return out
