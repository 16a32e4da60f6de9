"""Device-side counterpart of the reference's lib/pose/hrnet/lib/utils/inference.py get_final_preds (import as
device.lib.pose.hrnet.lib.utils.inference): argmax, the quarter-pixel shift and the inverse affine of every heatmap
in one launch (gast_b200.keypoints2d, DESIGN.md §8.6).  numpy heatmaps in -> numpy out (through the device), CUDA
tensor in -> CUDA tensors out without waiting for the device, so gen_kpts.py can drop `.clone().cpu().numpy()`.
Bit for bit the reference's when cv2 is importable (the inverse matrices come from cv2.getAffineTransform; without
cv2 they are only within a few ulps of it).
"""
import numpy as np
import torch

from gast_b200 import keypoints2d as _K
from gast_b200.engine import GastError

__all__ = ['get_final_preds']


def get_final_preds(config, batch_heatmaps, center, scale):
    """inference.py:48-82: preds (n, J, 2) float32 in frame pixels and maxvals (n, J, 1) float32 of batch_heatmaps
    (n, J, hh, hw) float32, with center and scale the (n, 2) float32 PreProcess returned; config.TEST.POST_PROCESS
    selects the quarter-pixel shift"""
    if isinstance(batch_heatmaps, torch.Tensor) and not batch_heatmaps.is_cuda:
        raise GastError('get_final_preds: the heatmaps must be a numpy array or a CUDA tensor')
    if len(batch_heatmaps.shape) != 4:
        raise GastError('get_final_preds: heatmaps (n, J, hh, hw) expected, got %s' % (tuple(batch_heatmaps.shape),))
    n, hh, hw = int(batch_heatmaps.shape[0]), int(batch_heatmaps.shape[2]), int(batch_heatmaps.shape[3])
    center = np.asarray(center, dtype=np.float32).reshape(-1, 2)
    scale = np.asarray(scale, dtype=np.float32).reshape(-1, 2)
    if center.shape[0] < n or scale.shape[0] < n:
        raise GastError('get_final_preds: %d heatmap records but %d centers and %d scales'
                        % (n, center.shape[0], scale.shape[0]))
    inv = np.stack([_K.inverse_matrix(center[i], scale[i], (hw, hh)) for i in range(n)]) if n else \
        np.zeros((0, 2, 3))
    preds, maxvals = _K.decode_heatmaps(batch_heatmaps, inv, bool(config.TEST.POST_PROCESS))
    if isinstance(batch_heatmaps, torch.Tensor):
        return preds, maxvals
    return preds.cpu().numpy(), maxvals.cpu().numpy()
