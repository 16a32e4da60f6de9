"""Whole-sequence inference with test-time augmentation, kept on the device (SURVEY.md §8f N1).

`evaluate_sequence` is what `reconstruction.evaluate` (reconstruction.py:148-170) / `main.evaluate`
(main.py:299-320, return_predictions) do around `model_pos(inputs_2d)`: edge-pad the keypoint
sequence by the model's padding, append the mirrored twin, run ONE forward on the (2, T+2*pad, J, 2)
batch, un-flip the twin and average -- here as two small CUDA kernels either side of the forward
instead of numpy on the host (common/generators.py:210-233) and torch indexing (main.py:314-318).
"""
import ctypes as C
import torch

from .engine import GastError, _cuda_f32, _ilist, _launch, refuse_half


def tta_prepare(seq, pad, causal_shift, kps_left, kps_right):
    """seq (T,J,F) CUDA float32 -> (2, T+2*pad, J, F)."""
    seq = _cuda_f32(seq, 'tta_prepare')
    T, J, F = (int(s) for s in seq.shape)
    out = torch.empty((2, T + 2 * pad, J, F), dtype=torch.float32, device=seq.device)
    kl, n = _ilist(kps_left)
    kr, _ = _ilist(kps_right)
    _launch(seq.device, 'gast_tta_prepare', C.c_void_p(seq.data_ptr()), C.c_void_p(out.data_ptr()), T, J, F, int(pad),
            int(causal_shift), n, kl, kr)
    return out


def tta_merge(pred, joints_left, joints_right):
    """pred (2,T,J,3) -> (T,J,3): mean of the prediction and the un-flipped prediction of the twin."""
    pred = _cuda_f32(pred, 'tta_merge')
    if pred.shape[0] != 2 or pred.shape[-1] != 3:
        raise GastError('tta_merge: (2,T,J,3) tensor expected')
    T, J = int(pred.shape[1]), int(pred.shape[2])
    out = torch.empty((T, J, 3), dtype=torch.float32, device=pred.device)
    jl, n = _ilist(joints_left)
    jr, _ = _ilist(joints_right)
    _launch(pred.device, 'gast_tta_merge', C.c_void_p(pred.data_ptr()), C.c_void_p(out.data_ptr()), T, J, n, jl, jr)
    return out


def evaluate_sequence(model_pos, keypoints, kps_left, kps_right, joints_left, joints_right, causal=False):
    """keypoints (T,J,2) (numpy or tensor, normalised screen coordinates) -> (T,J,3) CUDA tensor."""
    refuse_half(model_pos, 'tta.evaluate_sequence', 'test-time augmentation')
    dev = next(model_pos.parameters()).device
    seq = torch.as_tensor(keypoints, dtype=torch.float32).to(dev)
    pad = (model_pos.receptive_field() - 1) // 2
    shift = pad if causal else 0
    model_pos.eval()
    with torch.no_grad():
        batch = tta_prepare(seq, pad, shift, kps_left, kps_right)
        pred = model_pos(batch)
        return tta_merge(pred, joints_left, joints_right)
