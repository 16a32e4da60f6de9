"""Device-side counterpart of the reference's lib/pose/hrnet/lib/utils/utilitys.py PreProcess (import as
device.lib.pose.hrnet.lib.utils.utilitys): the pose net's input crops warped, scaled and normalised on the device
(gast_b200.keypoints2d, DESIGN.md §8.6), bit for bit the reference's when cv2 is importable (the crop matrices come
from cv2.getAffineTransform; without cv2 they are only within a few ulps of it, see gast_b200.keypoints2d).
"""
import numpy as np
import torch

from gast_b200 import keypoints2d as _K
from gast_b200.engine import GastError
from gast_b200.keypoints2d import box_to_center_scale  # noqa: F401  (the reference module's helper)

__all__ = ['PreProcess', 'box_to_center_scale']


def PreProcess(image, bboxs, cfg, num_pos=2):
    """utilitys.py:140-170: (inputs, image, centers, scales) for the first num_pos boxes of bboxs (x1, y1, x2, y2)
    on image (H, W, 3) uint8 BGR -- a numpy array, a CUDA tensor or a path cv2 reads.  inputs (n, 3, h, w) float32
    is a CUDA tensor in the reference's plane order (the caller's inputs[:, [2, 1, 0]] and .cuda() still apply);
    centers and scales are lists of float32 (2,) arrays."""
    if isinstance(image, str):
        import cv2
        image = cv2.imread(image, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
    if isinstance(image, torch.Tensor) and not image.is_cuda:
        raise GastError('PreProcess: the image must be a numpy array or a CUDA tensor')
    if len(image.shape) != 3 or image.shape[2] != 3:
        raise GastError('PreProcess: an (H, W, 3) image expected, got %s' % (tuple(image.shape),))
    H, W = int(image.shape[0]), int(image.shape[1])
    size = (int(cfg.MODEL.IMAGE_SIZE[0]), int(cfg.MODEL.IMAGE_SIZE[1]))
    centers, scales, mats = [], [], []
    for bbox in bboxs[:num_pos]:
        c, s = _K.center_scale(bbox, H, W)
        centers.append(c)
        scales.append(s)
        mats.append(_K.affine_pair(c, s, size)[0])
    if not mats:
        raise GastError('PreProcess: no boxes')
    frames = image.unsqueeze(0) if isinstance(image, torch.Tensor) else np.asarray(image)[None]
    inputs = _K.crop_persons(frames, np.zeros(len(mats), np.int64), np.stack(mats), size, net_order=False)
    return inputs, image, centers, scales
