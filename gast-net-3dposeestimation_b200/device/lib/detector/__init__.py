"""Device-side counterpart of the reference's lib/detector (import as device.lib.detector): yolo_human_det with the
letterbox and the post-processing on the device (gast_b200.detection, DESIGN.md §8.7).  Darknet itself, and
load_model, stay the reference's: load_model is imported from its lib.detector when first called."""
import numpy as np
import torch

from gast_b200 import detection as _D

__all__ = ['yolo_human_det', 'load_model']


def load_model(*args, **kwargs):
    """the reference's lib.detector.load_model (Darknet with its weights)"""
    from lib.detector import load_model as _load
    return _load(*args, **kwargs)


def yolo_human_det(img, model=None, reso=416, confidence=0.70, nms_thresh=0.4):
    """human_detector.py:106-157: (bboxs (n, 4) float32 in frame pixels rounded to 2 decimals, scores (n, 1) float32)
    as numpy arrays, or (None, None) without a person.  img: a (H, W, 3) uint8 BGR frame (numpy or CUDA) or an image
    path; model: the caller's Darknet (loaded with load_model(inp_dim=reso) when None).  nms_thresh replaces the
    reference's --nms-thresh from sys.argv.  The boxes come back to the host in one copy."""
    from .yolov3.preprocess import prep_image
    if model is None:
        model = load_model(inp_dim=reso)
    x, orig, (W, H) = prep_image(img, reso)
    with torch.no_grad():
        pred = model(x, True)
    N = int(pred.shape[1])
    boxes, scores, counts = _D.person_boxes(pred, (W, H), reso, confidence, nms_thresh, N)
    T = boxes.shape[0]
    packed = torch.cat([boxes.view(T, -1), scores.view(T, -1), counts.view(torch.float32).view(T, 1)], 1)
    packed = packed[0].cpu().numpy()
    n = int(packed[-1:].copy().view(np.int32)[0])
    if n == 0:
        return None, None
    bboxs = packed[:4 * N].reshape(N, 4)[:n].copy()
    sc = packed[4 * N:5 * N][:n].copy()[:, None]
    return bboxs, sc
