"""Device-side counterpart of the reference's tools/preprocess.py (import as device.tools.preprocess): the video
demo's COCO -> H36M keypoints and scores, low-confidence limb repair, and placement of the lifted persons in one
frame with the height rebased (csrc/pipeline.cuh; float32 in the reference's order of operations, bit-identical for
float32 input).  Same names, signatures and return structure.  numpy in -> numpy out (through the device), CUDA
tensor in -> CUDA tensor out; a CPU tensor raises.

`valid_frames` is the reference's list of per-person frame index arrays, or a list of CUDA int64 index tensors (what
`h36m_coco_format` returns for CUDA input).  Host syncs: `h36m_coco_format` reads the persons' keep flags and valid
frame counts back in one copy, because its output shapes depend on them.  `revise_kpts`, `revise_skes` and
`revise_skes_real_time` on CUDA inputs do not wait for the device.
"""
import json

import numpy as np
import torch

from gast_b200 import pipeline as _P
from gast_b200.engine import GastError

num_person = 2
num_joints = 17
ratio_2d_3d = 500.


def _is_cuda(x):
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise GastError('a CUDA tensor is required (there is no CPU path)')
        return True
    return False


def _dev_f32(x):
    """numpy / list -> CUDA float32 (a blocking upload: the numpy path returns numpy anyway)"""
    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).cuda()


def _upload(a, dev):
    """host array -> device without waiting for the device: staged through pinned memory"""
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(dev, non_blocking=True)


class _Frames(object):
    """valid_frames on the device: packed int64 frames, host offsets, and the (P,T) int32 mask; `host` keeps the host
    lists when they were given so"""

    def __init__(self, valid_frames, P, T, dev):
        if len(valid_frames) != P:
            raise ValueError('valid_frames has %d entries for %d persons' % (len(valid_frames), P))
        counts = [int(f.shape[0]) if isinstance(f, torch.Tensor) else int(np.asarray(f).reshape(-1).shape[0])
                  for f in valid_frames]
        self.offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        if all(_is_cuda(f) for f in valid_frames) and P > 0:
            self.host = None
            self.frames = torch.cat([f.reshape(-1).to(torch.int64) for f in valid_frames])
            self.mask = torch.zeros((P, T), dtype=torch.int32, device=dev)
            for p, f in enumerate(valid_frames):
                self.mask[p].index_fill_(0, f.reshape(-1).to(torch.int64), 1)
        else:
            self.host = [np.asarray(f, dtype=np.int64).reshape(-1) for f in valid_frames]
            packed = np.concatenate(self.host) if self.host else np.zeros(0, np.int64)
            if packed.size and (packed.min() < 0 or packed.max() >= T):
                raise IndexError('valid_frames index out of range for %d frames' % T)
            mask = np.zeros((P, T), np.int32)
            for p, f in enumerate(self.host):
                mask[p, f] = 1
            self.frames = _upload(packed, dev)
            self.mask = _upload(mask, dev)


def load_json(file_path):
    """The detector's keypoint JSON -> (keypoints (2,T,17,2), scores (2,T,17), label, label_index), parsed on the
    host as the reference does (preprocess.py:15-44): the first num_person skeletons with a bounding box per frame."""
    with open(file_path, 'r') as f:
        info = json.load(f)
    T = info['data'][-1]['frame_index']
    keypoints = np.zeros((num_person, T, num_joints, 2), dtype=np.float32)
    scores = np.zeros((num_person, T, num_joints), dtype=np.float32)
    for fr in info['data']:
        t = fr['frame_index'] - 1
        for p, sk in enumerate(fr['skeleton'][:num_person]):
            if len(sk['bbox']) == 0:
                continue
            keypoints[p, t] = np.asarray(sk['pose'], dtype=np.float32)
            scores[p, t] = np.asarray(sk['score'], dtype=np.float32).reshape(-1)
    return keypoints, scores, info['label'], info['label_index']


def h36m_coco_format(keypoints, scores):
    """(P,T,17,2) COCO keypoints, (P,T,17) scores -> (H36M keypoints (K,T,17,2), H36M scores (K,T,17), valid_frames)
    of the K slots that hold a person (some coordinate non-zero).  One host sync: the keep flags and frame counts."""
    assert len(keypoints.shape) == 4 and len(scores.shape) == 3
    on_dev = _is_cuda(keypoints)
    if _is_cuda(scores) != on_dev:
        raise GastError('h36m_coco_format: keypoints and scores must both be CUDA tensors or both host arrays')
    k = keypoints if on_dev else _dev_f32(keypoints)
    s = scores if on_dev else _dev_f32(scores)
    out, sout, valid, keep = _P.h36m_coco_format(k, s)
    flags = torch.cat([keep, valid.sum(1, dtype=torch.int32)]).cpu().numpy()       # the one sync
    P = int(keep.shape[0])
    kept = [p for p in range(P) if flags[p]]
    if not on_dev:
        out, sout, valid = out.cpu().numpy(), sout.cpu().numpy(), valid.cpu().numpy()
        frames = [np.where(valid[p] != 0)[0] for p in kept]
        if not kept:                                          # np.asarray([]) of the reference
            return np.zeros((0,), np.float32), np.zeros((0,), np.float32), frames
        return out[kept], sout[kept], frames
    frames = [torch.nonzero_static(valid[p], size=int(flags[P + p])).reshape(-1) for p in kept]
    if not kept:
        e = torch.zeros((0,), dtype=torch.float32, device=k.device)
        return e, e.clone(), frames
    idx = torch.tensor(kept, dtype=torch.int64).to(k.device, non_blocking=True)
    return out.index_select(0, idx), sout.index_select(0, idx), frames


def revise_kpts(h36m_kpts, h36m_scores, valid_frames):
    """(P,T,J,2) keypoints, (P,T,J) scores, valid_frames -> (P,T,J,2): zero outside each person's valid frames, the
    low-confidence limb joints repaired at them (preprocess.py:78-112)."""
    on_dev = _is_cuda(h36m_kpts)
    k = h36m_kpts if on_dev else _dev_f32(h36m_kpts)
    s = (h36m_scores if _is_cuda(h36m_scores) else _dev_f32(h36m_scores).to(k.device))
    fr = _Frames(valid_frames, int(k.shape[0]), int(k.shape[1]), k.device)
    out = _P.revise_kpts(k, s, fr.mask)
    return out if on_dev else out.cpu().numpy()


def load_kpts_json(kpts_json):
    """-> (re_kpts, valid_frames, scores, label, label_index) as numpy, as the reference returns them: the JSON is
    parsed on the host, the keypoints converted and repaired on the device."""
    keypoints, scores, label, label_index = load_json(kpts_json)
    h36m_kpts, h36m_scores, valid_frames = h36m_coco_format(keypoints, scores)
    re_kpts = revise_kpts(h36m_kpts, h36m_scores, valid_frames)
    return re_kpts, valid_frames, scores, label, label_index


def revise_skes(prediction, re_kpts, valid_frames):
    """prediction: per person (F_p, J, 3) poses of its valid frames; re_kpts (P,T,J,2) -> (P,T,J,3) in one shared frame
    with the height rebased (preprocess.py:123-155).  Two persons without a common valid frame raise ValueError as in
    the reference when the frames are host arrays; with CUDA index tensors that check would need a host read, so their
    x and y come out NaN instead."""
    on_dev = _is_cuda(re_kpts)
    k = re_kpts if on_dev else _dev_f32(re_kpts)
    P, T = int(k.shape[0]), int(k.shape[1])
    fr = _Frames(valid_frames, P, T, k.device)
    if fr.host is not None and P == 2 and np.intersect1d(fr.host[0], fr.host[1]).size == 0 \
            and max(fr.host[0].size, fr.host[1].size) > 0:
        raise ValueError('revise_skes: the two persons share no valid frame')
    if len(prediction) != P:
        raise ValueError('revise_skes: %d predictions for %d persons' % (len(prediction), P))
    preds = [p if _is_cuda(p) else _dev_f32(p).to(k.device) for p in prediction]
    for p, (a, b) in enumerate(zip(preds, np.diff(fr.offsets))):
        if int(a.shape[0]) != int(b):
            raise ValueError('revise_skes: person %d has %d poses for %d valid frames' % (p, int(a.shape[0]), int(b)))
    pred = torch.cat([p.reshape(-1, int(k.shape[2]), 3) for p in preds]).to(torch.float32)
    out = _P.revise_skes(pred, fr.frames, fr.offsets, k)
    return out if on_dev else out.cpu().numpy()


def revise_skes_real_time(prediction, re_kpts, width):
    """prediction (M,17,3) poses and re_kpts (M,17,2) keypoints of one tick -> (M,17,3) placed by each person's image
    position, height rebased over all M (preprocess.py:158-172)."""
    if isinstance(prediction, (list, tuple)):
        prediction = torch.stack(list(prediction)) if prediction and _is_cuda(prediction[0]) else np.stack(prediction)
    on_dev = _is_cuda(prediction)
    pr = prediction if on_dev else _dev_f32(prediction)
    k = re_kpts if _is_cuda(re_kpts) else _dev_f32(re_kpts).to(pr.device)
    out = _P.revise_skes_real_time(pr, k, width)
    return out if on_dev else out.cpu().numpy()
