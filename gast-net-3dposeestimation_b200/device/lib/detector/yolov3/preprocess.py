"""Device-side counterpart of the reference's lib/detector/yolov3/preprocess.py prep_image (import as
device.lib.detector.yolov3.preprocess): the letterbox, BGR -> RGB and /255 in one launch (gast_b200.detection,
DESIGN.md §8.7), bit for bit OpenCV's own INTER_CUBIC resize.  The network input comes back as a CUDA tensor.
"""
import numpy as np
import torch

from gast_b200 import detection as _D
from gast_b200.engine import GastError

__all__ = ['prep_image']


def prep_image(img, inp_dim):
    """preprocess.py:24-38: (img_ (1, 3, inp_dim, inp_dim) float32 CUDA tensor, orig_im, (W, H)) for a (H, W, 3)
    uint8 BGR frame (numpy or CUDA) or an image path (read with cv2, as the reference does)"""
    if isinstance(img, str):
        import cv2
        orig_im = cv2.imread(img)
        if orig_im is None:
            raise GastError('prep_image: cannot read %s' % img)
    else:
        orig_im = img
    if len(orig_im.shape) != 3:
        raise GastError('prep_image: a (H, W, 3) frame expected, got %s' % (tuple(orig_im.shape),))
    dim = int(orig_im.shape[1]), int(orig_im.shape[0])
    frames = orig_im[None] if isinstance(orig_im, torch.Tensor) else np.asarray(orig_im)[None]
    return _D.letterbox(frames, inp_dim), orig_im, dim
