"""Device-side counterpart of the reference's lib/detector/yolov3/util.py write_results (import as
device.lib.detector.yolov3.util): the confidence mask, corners, class argmax, person filter, sort and greedy NMS of
every image in one launch (gast_b200.detection, DESIGN.md §8.7).  Only det_hm=True (the person detector's call) is
served.  The output's row count depends on the data, so it reads the counts back once.
"""
import torch

from gast_b200 import detection as _D
from gast_b200.engine import GastError

__all__ = ['write_results']


def write_results(prediction, confidence, num_classes, nms=True, nms_conf=0.4, det_hm=False):
    """util.py:107-225 with det_hm=True: Num_obj x [img_index, x1, y1, x2, y2, objectness, class score, 0] float32
    on the device, image by image, each image's rows objectness descending after NMS (exact ties: the lower prediction
    index first), the corners in the network input's pixels.

    Kept bug for bug: with more than one image, the first image that has no row of the person class ends the call,
    which then returns that image's empty (0, 7) selection and drops the rows of the images before it."""
    if not det_hm:
        raise GastError('write_results: only det_hm=True (the person detector) runs on the device')
    if not nms:
        raise GastError('write_results: only nms=True runs on the device')
    if int(num_classes) != 80:
        raise GastError('write_results: 80 classes expected, got %d' % int(num_classes))
    if not isinstance(prediction, torch.Tensor) or not prediction.is_cuda or prediction.dim() != 3:
        raise GastError('write_results: prediction must be a (B, N, 85) CUDA tensor')
    B, N = int(prediction.shape[0]), int(prediction.shape[1])
    D = next((d for d in range(64, 641, 32) if _D.num_predictions(d) == N), None)
    if D is None:
        raise GastError('write_results: %d predictions match no input size' % N)
    boxes, scores, counts, mconf, persons = _D.person_boxes(prediction, (D, D), D, confidence, nms_conf, N, raw=True,
                                                            extras=True)
    host = torch.stack([counts, persons], 1).cpu()
    rows = []
    for b in range(B):
        if int(host[b, 1]) == 0:
            return prediction.new_empty((0, 7))
        n = int(host[b, 0])
        ind = prediction.new_full((n, 1), float(b))
        rows.append(torch.cat([ind, boxes[b, :n], scores[b, :n, None], mconf[b, :n, None],
                               torch.zeros_like(ind)], 1))
    return torch.cat(rows) if rows else prediction.new_empty((0, 8))
