"""The person detector's letterbox and post-processing on the device (lib/detector/yolov3/human_detector.py:106-157).

`letterbox` is preprocess.prep_image (letterbox_image's cv2.resize(INTER_CUBIC) into a 128 canvas, BGR -> RGB, /255)
for any number of frames in one launch; `person_boxes` is write_results(det_hm=True) plus yolo_human_det's rescale,
clamp and round(v, 2) for any number of frames in one launch.  Both take numpy arrays or CUDA tensors, return CUDA
tensors and do not wait for the device.  `video_boxes` is the front half of gen_video_kpts on a chunk of decoded
frames: one letterbox launch, one call to the caller's Darknet, one post-processing launch, one copy to the host, then
the caller's tracker frame by frame (or, with a tracking.DeviceSort, one tracking launch before the copy).  The kernels are csrc/detect.cuh; every formula is in DESIGN.md §8.7.

The letterbox equals OpenCV's own INTER_CUBIC resize bit for bit; cv2 builds that route the resize through IPP differ
from it by at most one grey level in a few percent of the bytes.  Exact objectness ties, which the reference's sort
leaves in no defined order, keep the lower prediction index first.

Refused before any launch (GastError): a frame side above 32767, a letterbox size of 0, an inp_dim that is not a
multiple of 32 above 32 or whose predictions do not fit one CTA's shared memory (above 640), predictions whose count is
not 3 * sum((inp_dim / s)^2) for s = 32, 16, 8 or whose last dimension is not 85, non-float32 predictions, and frame
sizes that do not match the predictions.
"""
import numpy as np
import torch

from .engine import GastError, _launch, _p
from .keypoints2d import _device, _on_device

MAX_SIDE = 32767
ATTRS = 85
STRIDES = (32, 16, 8)
MAX_SMEM = 227 * 1024          # one CTA per frame holds 9 bytes per prediction
MAX_DET = 100
RGB_INPUT = 1                  # gast_letterbox flag
RAW = 1                        # gast_person_detections flag


def num_predictions(inp_dim):
    """Darknet's rows for inp_dim: 3 anchors on each of the 32, 16 and 8 strides"""
    return 3 * sum((inp_dim // s) ** 2 for s in STRIDES)


def check_inp_dim(inp_dim):
    D = int(inp_dim)
    if D <= 32 or D % 32:
        raise GastError('detection: inp_dim %d (a multiple of 32 above 32, as load_model asserts)' % D)
    if 9 * num_predictions(D) > MAX_SMEM:
        raise GastError('detection: inp_dim %d: %d predictions do not fit one CTA\'s shared memory (inp_dim <= 640)'
                        % (D, num_predictions(D)))
    return D


def letterbox_geometry(W, H, inp_dim):
    """(new_w, new_h): letterbox_image's expression in double, as written"""
    new_w = int(W * min(inp_dim / W, inp_dim / H))
    new_h = int(H * min(inp_dim / W, inp_dim / H))
    return new_w, new_h


def letterbox(frames, inp_dim=416, rgb_input=False):
    """prep_image's network input (F, 3, D, D) float32 RGB planes on the device for frames (F, H, W, 3) uint8 (BGR as
    cv2 reads them, RGB with rgb_input), numpy or CUDA, bit for bit OpenCV's own INTER_CUBIC path"""
    dtype = frames.dtype if isinstance(frames, torch.Tensor) else np.asarray(frames).dtype
    if dtype not in (torch.uint8, np.uint8):
        raise GastError('detection: frames must be uint8, got %s' % dtype)
    shape = tuple(frames.shape)
    if len(shape) != 4 or shape[-1] != 3:
        raise GastError('detection: frames (F, H, W, 3) expected, got %s' % (shape,))
    F, H, W = int(shape[0]), int(shape[1]), int(shape[2])
    if not (0 < H <= MAX_SIDE and 0 < W <= MAX_SIDE):
        raise GastError('detection: a %d x %d frame (each side 1 .. %d)' % (W, H, MAX_SIDE))
    D = int(inp_dim)
    if D <= 32 or D % 32:
        raise GastError('detection: inp_dim %d (a multiple of 32 above 32, as load_model asserts)' % D)
    nw, nh = letterbox_geometry(W, H, D)
    if nw <= 0 or nh <= 0:
        raise GastError('detection: a %d x %d frame letterboxes to %d x %d' % (W, H, nw, nh))
    dev = frames.device if isinstance(frames, torch.Tensor) and frames.is_cuda else _device(None)
    out = torch.empty((F, 3, D, D), dtype=torch.float32, device=dev)
    if F:
        fr = _on_device(frames, torch.uint8, dev, 'frames')
        _launch(dev, 'gast_letterbox', _p(fr), F, H, W, D, nw, nh, RGB_INPUT if rgb_input else 0, _p(out))
    return out


def _frame_sizes(frame_sizes, F, dev):
    if isinstance(frame_sizes, torch.Tensor) and frame_sizes.is_cuda:
        s = frame_sizes.to(device=dev, dtype=torch.int32).contiguous().view(-1, 2)
    else:
        a = np.asarray(frame_sizes, dtype=np.int64).reshape(-1, 2)
        if a.shape[0] == 1 and F > 1:
            a = np.repeat(a, F, 0)
        if a.size and (a.min() <= 0 or a.max() > MAX_SIDE):
            raise GastError('detection: frame sizes outside 1 .. %d' % MAX_SIDE)
        s = _on_device(a, torch.int32, dev, 'frame_sizes')
    if int(s.shape[0]) != F:
        raise GastError('detection: %d frames of predictions but %d frame sizes' % (F, int(s.shape[0])))
    return s


def person_boxes(predictions, frame_sizes, inp_dim=416, confidence=0.7, nms_thresh=0.4, max_det=MAX_DET,
                 raw=False, extras=False):
    """yolo_human_det's boxes and scores for every frame of predictions (F, N, 85) float32 (Darknet.forward's output
    for a batch of letterboxed frames), numpy or CUDA.  frame_sizes: (F, 2) or one (W, H) for all frames.

    Returns boxes (F, max_det, 4) float32 in frame pixels rounded as round(v, 2), scores (F, max_det) float32 (the
    objectness) in the reference's order (objectness descending after NMS; ties: lower prediction index first), zero
    past the count, and counts (F,) int32, the true number of survivors (it may exceed max_det); all on the device.
    raw=True leaves the boxes as write_results' corners in the D x D input.  extras=True also returns write_results'
    class-score column (F, max_det) and the number of rows that reach its person filter (F,) int32."""
    if isinstance(predictions, torch.Tensor):
        if predictions.dtype != torch.float32:
            raise GastError('detection: predictions must be float32, got %s' % predictions.dtype)
    elif np.asarray(predictions).dtype != np.float32:
        raise GastError('detection: predictions must be float32, got %s' % np.asarray(predictions).dtype)
    shape = tuple(predictions.shape)
    D = check_inp_dim(inp_dim)
    if len(shape) != 3 or shape[2] != ATTRS:
        raise GastError('detection: predictions (F, N, 85) expected, got %s' % (shape,))
    F, N = int(shape[0]), int(shape[1])
    if N != num_predictions(D):
        raise GastError('detection: %d predictions per frame for inp_dim %d (%d expected)' % (N, D, num_predictions(D)))
    K = int(max_det)
    if K < 0:
        raise GastError('detection: max_det must be >= 0')
    dev = predictions.device if isinstance(predictions, torch.Tensor) and predictions.is_cuda else _device(None)
    sizes = _frame_sizes(frame_sizes, F, dev)
    boxes = torch.empty((F, K, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((F, K), dtype=torch.float32, device=dev)
    counts = torch.empty(F, dtype=torch.int32, device=dev)
    mconf = torch.empty((F, K), dtype=torch.float32, device=dev) if extras else None
    persons = torch.empty(F, dtype=torch.int32, device=dev) if extras else None
    if F:
        pred = _on_device(predictions, torch.float32, dev, 'predictions')
        _launch(dev, 'gast_person_detections', _p(pred), F, N, ATTRS, D, _p(sizes), float(np.float32(confidence)),
                float(np.float32(nms_thresh)), K, RAW if raw else 0, _p(boxes), _p(scores), _p(counts), _p(mconf),
                _p(persons))
    if extras:
        return boxes, scores, counts, mconf, persons
    return boxes, scores, counts


def video_boxes(frames, det_net, tracker, inp_dim=416, confidence=0.7, nms_thresh=0.4, max_det=MAX_DET,
                rgb_input=False, on_device=False):
    """The front half of gen_video_kpts (gen_kpts.py:199-227) on a chunk of decoded frames (T, H, W, 3) uint8 (BGR
    as cv2 reads them, RGB with rgb_input), numpy or CUDA.

    det_net(batch, True) is the caller's Darknet: (T, 3, D, D) float32 letterboxed frames on the device to (T, N, 85)
    predictions on the device.  One letterbox launch, one net call, one post-processing launch and one copy of the
    boxes and counts to the host; then tracker.update(bboxs) (the reference's Sort) for each frame in order with
    yolo_human_det's (n, 4) float32 boxes, skipping frames without a box or whose boxes are all zero.  A
    gast_b200.tracking.DeviceSort tracker runs on the device instead, in one launch after the post-processing, and
    the chunk's one copy is of its tracks.

    Returns the T per-frame tracker outputs, None for a skipped frame: what video_keypoints takes as boxes.  Raises
    GastError if a frame has more than max_det boxes.  With a DeviceSort and on_device=True nothing is copied: it
    returns update_chunk's (rows, counts, status) on the device, which video_keypoints also takes as boxes, so the
    chain to the keypoints makes no per-box host work."""
    from .tracking import DeviceSort, host_tracks
    if on_device and not isinstance(tracker, DeviceSort):
        raise GastError('detection: on_device=True needs a tracking.DeviceSort tracker')
    shape = tuple(frames.shape)
    if len(shape) != 4 or shape[-1] != 3:
        raise GastError('detection: frames (T, H, W, 3) expected, got %s' % (shape,))
    T, H, W = int(shape[0]), int(shape[1]), int(shape[2])
    if T == 0:
        if on_device:
            return tracker.update_chunk(np.zeros((0, max_det, 4), np.float32), np.zeros(0, np.int32))
        return []
    D = check_inp_dim(inp_dim)
    batch = letterbox(frames, D, rgb_input=rgb_input)
    with torch.no_grad():
        pred = det_net(batch, True)
    if not isinstance(pred, torch.Tensor) or not pred.is_cuda or tuple(pred.shape) != (T, num_predictions(D), ATTRS):
        raise GastError('detection: the detector must return (%d, %d, %d) predictions on the device'
                        % (T, num_predictions(D), ATTRS))
    boxes, _, counts = person_boxes(pred, (W, H), D, confidence, nms_thresh, max_det)
    if isinstance(tracker, DeviceSort):
        # the tracker on the device too: the chunk's one copy is of the tracks, or none with on_device
        tracks = tracker.update_chunk(boxes, counts, skip_empty=True)
        return tracks if on_device else host_tracks(*tracks)
    # one copy: the boxes and the counts' bits side by side
    packed = torch.cat([boxes.view(T, -1), counts.view(torch.float32).view(T, 1)], 1).cpu().numpy()
    counts = packed[:, -1].copy().view(np.int32)
    boxes = packed[:, :-1].reshape(T, max_det, 4)
    if counts.max() > max_det:
        raise GastError('detection: a frame has %d boxes (max_det = %d)' % (int(counts.max()), max_det))
    out = []
    for t in range(T):
        bboxs = boxes[t, :counts[t]]
        if counts[t] == 0 or not bboxs.any():
            out.append(None)
            continue
        out.append(tracker.update(bboxs.copy()))
    return out
