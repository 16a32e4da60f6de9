"""Device-side counterpart of the reference's tools/inference.py (import as device.tools.inference): the video demo's
lifting of each person's keypoints with test-time augmentation and the demo's fixed camera rotation, on the device.
Same names, signatures and return structure: numpy in -> numpy out, CUDA tensor in -> CUDA tensor out.

Per person: normalize_screen_coordinates -> edge padding by the caller's `pad` / `causal_shift` plus the mirrored
twin (gast_tta_prepare) -> model_pos -> un-flip and average (gast_tta_merge) -> camera_to_world(rot).  The padding is
the caller's, as in the reference, not the model's own.
"""
import numpy as np
import torch

from gast_b200 import pipeline as _P
from gast_b200 import tta as _T
from gast_b200.engine import GastError

joints_left, joints_right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
kps_left, kps_right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
rot = np.array([0.14070565, -0.15007018, -0.7552408, 0.62232804], dtype=np.float32)


def _is_cuda(x):
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            raise GastError('a CUDA tensor is required (there is no CPU path)')
        return True
    return False


def _model_device(model_pos):
    return next(model_pos.parameters()).device


def evaluate(test_generator, model_pos):
    """One (T,J,3) prediction per sequence of `test_generator` (the reference's or device.common.generators'
    UnchunkedGenerator), the augmented twin un-flipped and averaged in.  CUDA batches -> CUDA tensors, numpy batches ->
    numpy arrays."""
    dev = _model_device(model_pos)
    prediction = []
    with torch.no_grad():
        for _, _, batch_2d in test_generator.next_epoch():
            on_dev = _is_cuda(batch_2d)
            x = batch_2d if on_dev else torch.as_tensor(np.ascontiguousarray(batch_2d, dtype=np.float32)).to(dev)
            pred = model_pos(x.to(torch.float32))
            if test_generator.augment_enabled():
                pred = _T.tta_merge(pred, joints_left, joints_right)
            else:
                pred = pred.squeeze(0)
            prediction.append(pred if on_dev else pred.cpu().numpy())
    return prediction


def _lift(seq, width, height, model_pos, pad, causal_shift):
    """(F,J,2) pixel keypoints on the device -> (F',J,3) world poses"""
    norm = _P.normalize_screen(seq, width, height)
    with torch.no_grad():
        batch = _T.tta_prepare(norm, int(pad), int(causal_shift), kps_left, kps_right)
        pred = _T.tta_merge(model_pos(batch), joints_left, joints_right)
    return _P.camera_to_world(pred, R=rot, t=0)


def _dev_f32(x, dev):
    return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float32)).to(dev)


def gen_pose(kpts, valid_frames, width, height, model_pos, pad, causal_shift=0):
    """kpts (P,T,17,2), valid_frames -> per person the (F_p,17,3) world poses of its valid frames."""
    assert len(kpts.shape) == 4, 'The shape of kpts: {}'.format(kpts.shape)
    assert kpts.shape[0] == len(valid_frames)
    on_dev = _is_cuda(kpts)
    k = kpts if on_dev else _dev_f32(kpts, _model_device(model_pos))
    out = []
    for p, frames in enumerate(valid_frames):
        idx = frames.reshape(-1).to(torch.int64) if _is_cuda(frames) else \
            torch.as_tensor(np.asarray(frames, dtype=np.int64).reshape(-1)).to(k.device)
        pose = _lift(k[p].index_select(0, idx).contiguous(), width, height, model_pos, pad, causal_shift)
        out.append(pose if on_dev else pose.cpu().numpy())
    return out


def _rebase(pose):
    """pose[..., 2] -= min over all of pose[..., 2]"""
    pose[..., 2] -= torch.amin(pose[..., 2])
    return pose


def gen_pose_frame(kpts, width, height, model_pos, pad, causal_shift=0):
    """kpts (M,T,17,2): M persons' windows -> per person the (17,3) world pose of the first output frame, height
    rebased per person."""
    on_dev = _is_cuda(kpts)
    k = kpts if on_dev else _dev_f32(kpts, _model_device(model_pos))
    out = []
    for m in range(int(k.shape[0])):
        pose = _rebase(_lift(k[m].contiguous(), width, height, model_pos, pad, causal_shift)[0])
        out.append(pose if on_dev else pose.cpu().numpy())
    return out


def gen_pose_frame_(kpts, width, height, model_pos, pad, causal_shift=0):
    """kpts (N,17,2+): one sequence -> (N',17,3) world poses, height rebased over the whole sequence."""
    if not isinstance(kpts, (np.ndarray, torch.Tensor)):
        kpts = np.array(kpts)
    on_dev = _is_cuda(kpts)
    k = kpts if on_dev else _dev_f32(kpts, _model_device(model_pos))
    pose = _rebase(_lift(k[..., :2].contiguous(), width, height, model_pos, pad, causal_shift))
    return pose if on_dev else pose.cpu().numpy()
