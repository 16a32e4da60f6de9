"""CPU restatement (numpy) of the steps either side of the lifting forward (SURVEY.md §8f N1-N3).

TEST INFRASTRUCTURE ONLY -- imported by tests/ (and nothing in the product path).  Pinned against
outputs of the unmodified reference generated in the build container (tests/golden/pipeline_17.npz,
tests/golden/make_golden.py::pipeline_cases); each function cites the reference lines it restates.
"""
import numpy as np

F32 = np.float32


# ---------------------------------------------------------------------------------------------
# common/generators.py:4-154  ChunkedGenerator
# ---------------------------------------------------------------------------------------------
def chunk_pairs(lengths, chunk_length, augment):
    """generators.py:31-41: (seq, start, end, flip) rows, per video the plain chunks then the flipped ones."""
    rows = []
    for i, n in enumerate(lengths):
        n_chunks = (n + chunk_length - 1) // chunk_length
        offset = (n_chunks * chunk_length - n) // 2
        starts = np.arange(n_chunks) * chunk_length - offset
        for flip in ((0, 1) if augment else (0,)):
            for s in starts:
                rows.append((i, s, s + chunk_length, flip))
    return np.array(rows, dtype=np.int64).reshape(-1, 4)


def _mirror(a, left, right):
    """generators.py:118-121 / 131-135: negate coordinate 0, swap the left and right joints."""
    perm = np.arange(a.shape[-2])
    perm[list(left)], perm[list(right)] = list(right), list(left)
    b = a[..., perm, :].copy()
    b[..., 0] = -b[..., 0]
    return b


def chunk_batch(poses_2d, poses_3d, cameras, pairs, chunk_length, pad, causal_shift, kps_left, kps_right, joints_left,
                joints_right):
    """generators.py:98-144 for one batch of `pairs`: windows with edge replication, optional mirroring."""
    b2, b3, bc = [], [], []
    for seq, start, _end, flip in np.asarray(pairs).reshape(-1, 4):
        s2 = poses_2d[seq]
        idx = np.clip(np.arange(start - pad - causal_shift, start + chunk_length + pad - causal_shift), 0, len(s2) - 1)
        w2 = s2[idx].astype(F32)
        b2.append(_mirror(w2, kps_left, kps_right) if flip else w2)
        if poses_3d is not None:
            s3 = poses_3d[seq]
            w3 = s3[np.clip(np.arange(start, start + chunk_length), 0, len(s3) - 1)].astype(F32)
            b3.append(_mirror(w3, joints_left, joints_right) if flip else w3)
        if cameras is not None:
            c = np.array(cameras[seq], dtype=F32)
            if flip:
                c[2], c[7] = -c[2], -c[7]                     # generators.py:141-144
            bc.append(c)
    return (np.stack(bc) if bc else None, np.stack(b3) if b3 else None, np.stack(b2))


# ---------------------------------------------------------------------------------------------
# tools/mpii_coco_h36m.py  (float32 throughout, sums left to right like numpy's reduction of <8 items)
# ---------------------------------------------------------------------------------------------
_COCO_TO_H36M = {9: 0, 11: 5, 14: 6, 12: 7, 15: 8, 13: 9, 16: 10, 4: 11, 1: 12, 5: 13, 2: 14, 6: 15, 3: 16}


def _valid(frames):
    return np.where(np.sum(frames.reshape(frames.shape[0], -1), axis=1) != 0)[0]


def coco_h36m(kp):
    """mpii_coco_h36m.py:20-48.  kp (T,17,2) float32 COCO order -> (T,17,2) Human3.6M order."""
    kp = np.asarray(kp, dtype=F32)
    out = np.zeros_like(kp)
    nose, l_sho, r_sho, l_hip, r_hip = kp[:, 0], kp[:, 5], kp[:, 6], kp[:, 11], kp[:, 12]
    sho_mid = (l_sho + r_sho) / F32(2)
    head = np.empty_like(nose)
    head[:, 0] = (((kp[:, 1, 0] + kp[:, 2, 0]) + kp[:, 3, 0]) + kp[:, 4, 0]) / F32(4)     # :25
    head[:, 1] = (kp[:, 1, 1] + kp[:, 2, 1]) - nose[:, 1]                                 # :26
    thorax = sho_mid + (nose - sho_mid) / F32(3)                                          # :27-28
    pelvis = (l_hip + r_hip) / F32(2)                                                     # :30
    spine = (((l_sho + r_sho) + l_hip) + r_hip) / F32(4)                                  # :31
    out[:, 10], out[:, 8], out[:, 0], out[:, 7] = head, thorax, pelvis, spine             # :33
    for h, c in _COCO_TO_H36M.items():                                                    # :34
        out[:, h] = kp[:, c]
    out[:, 9] = out[:, 9] - (out[:, 9] - sho_mid) / F32(4)                                # :36
    out[:, 7, 0] = out[:, 7, 0] + F32(2) * (out[:, 7, 0] - (out[:, 0, 0] + out[:, 8, 0]) / F32(2))   # :37
    eye_mid_y = (kp[:, 1, 1] + kp[:, 2, 1]) / F32(2)
    out[:, 8, 1] = out[:, 8, 1] - (eye_mid_y - nose[:, 1]) * F32(2) / F32(3)              # :38
    return out, _valid(out)


def mpii_h36m(kp):
    """mpii_coco_h36m.py:51-59.  (T,16,2) -> (T,17,2)."""
    kp = np.asarray(kp, dtype=F32)
    order = [3, 2, 1, 4, 5, 6, 0, 8, 9, 10, 16, 15, 14, 11, 12, 13]
    out = np.zeros((kp.shape[0], 17, 2), F32)
    out[:, order] = kp
    out[:, 7] = (((kp[:, 2] + kp[:, 3]) + kp[:, 12]) + kp[:, 13]) / F32(4)
    return out, _valid(out)


def coco_h36m_toe_format(kp):
    """mpii_coco_h36m.py:62-78.  COCO whole-body (T,>=22,2) -> (T,19,2) body + toes."""
    kp = np.asarray(kp, dtype=F32)
    body, _ = coco_h36m(kp[:, :17])
    out = np.zeros((kp.shape[0], 19, 2), F32)
    out[:, [0, 1, 2, 3, 5, 6, 7, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18]] = body
    out[:, 4] = (kp[:, 20] + kp[:, 21]) / F32(2)
    out[:, 8] = (kp[:, 17] + kp[:, 18]) / F32(2)
    return out, _valid(out)


# ---------------------------------------------------------------------------------------------
# common/camera.py:8-28, common/quaternion.py:4-18
# ---------------------------------------------------------------------------------------------
def normalize_screen_coordinates(X, w, h):
    """camera.py:8-12: float32 X/w*2, then minus the float64 pair [1, h/w]; callers cast to float32."""
    s = (np.asarray(X, F32) / F32(w)) * F32(2)
    return (s.astype(np.float64) - np.array([1.0, h / w])).astype(F32)


def image_coordinates(X, w, h):
    """camera.py:15-19."""
    return ((np.asarray(X, F32).astype(np.float64) + np.array([1.0, h / w])) * w / 2).astype(F32)


def camera_to_world(X, R, t=0):
    """camera.py:27-28 with quaternion.py:4-18: v + 2 (q0 (qv x v) + qv x (qv x v)) + t."""
    v = np.asarray(X, np.float64)
    q = np.asarray(R, np.float64)
    qv = np.broadcast_to(q[1:], v.shape)
    uv = np.cross(qv, v)
    uuv = np.cross(qv, uv)
    return (v + 2 * (q[0] * uv + uuv) + t).astype(F32)


# ---------------------------------------------------------------------------------------------
# common/loss.py:5-53
# ---------------------------------------------------------------------------------------------
def mpjpe(pred, tgt):
    """loss.py:5-11 and its gradient w.r.t. pred (0 where the distance is 0, as torch.norm's backward)."""
    d = np.asarray(pred, np.float64) - np.asarray(tgt, np.float64)
    nrm = np.sqrt((d * d).sum(-1, keepdims=True))
    n = nrm.size
    with np.errstate(invalid='ignore', divide='ignore'):
        g = np.where(nrm > 0, d / nrm, 0.0) / n
    return nrm.mean(), g


def p_mpjpe_per_frame(pred, tgt):
    """loss.py:14-53 frame by frame (float64): Procrustes (scale, rotation, translation) then mean distance.  A frame
    with zero spread gives NaN (loss.py:30-31 divide by its zero norm; numpy's SVD then raises on the NaN matrix)."""
    out = []
    for Y, X in zip(np.asarray(pred, np.float64), np.asarray(tgt, np.float64)):
        muX, muY = X.mean(0), Y.mean(0)
        X0, Y0 = X - muX, Y - muY
        nX, nY = np.sqrt((X0 ** 2).sum()), np.sqrt((Y0 ** 2).sum())
        if nX == 0 or nY == 0:
            out.append(np.nan)
            continue
        U, s, Vt = np.linalg.svd((X0 / nX).T @ (Y0 / nY))
        V = Vt.T
        if np.linalg.det(V @ U.T) < 0:                                   # :39-43
            V[:, -1] *= -1
            s[-1] *= -1
        R = V @ U.T
        a = s.sum() * nX / nY
        aligned = a * Y @ R + (muX - a * muY @ R)
        out.append(np.linalg.norm(aligned - X, axis=-1).mean())
    return np.array(out)


def adam_step(p, g, m, v, vmax, step, lr, b1=0.9, b2=0.999, eps=1e-8, weight_decay=0.0, amsgrad=True):
    """torch/optim/adam.py single-tensor update, in place, float64; amsgrad=True is what trainval.py:78 constructs.
    weight_decay adds weight_decay * p to the gradient (L2, not decoupled); vmax is unused without amsgrad."""
    if weight_decay != 0:
        g = g + weight_decay * p
    m[:] = m + (1 - b1) * (g - m)
    v[:] = b2 * v + (1 - b2) * g * g
    if amsgrad:
        np.maximum(vmax, v, out=vmax)
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    p[:] = p - (lr / bc1) * m / (np.sqrt(vmax if amsgrad else v) / np.sqrt(bc2) + eps)


def adam_amsgrad_step(p, g, m, v, vmax, step, lr, b1=0.9, b2=0.999, eps=1e-8):
    """adam_step with amsgrad=True and no weight decay: what trainval.py:78 constructs."""
    adam_step(p, g, m, v, vmax, step, lr, b1, b2, eps)
