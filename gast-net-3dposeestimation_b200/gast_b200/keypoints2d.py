"""The 2D pose net's input crops and heatmap decode on the device (lib/pose/hrnet/pose_estimation/gen_kpts.py:234-256).

`crop_persons` is PreProcess's warp, ToTensor and Normalize (lib/pose/hrnet/lib/utils/utilitys.py:140-170) for any
number of boxes of any number of frames in one launch; `decode_heatmaps` is get_final_preds
(lib/pose/hrnet/lib/utils/inference.py:21-82) in one launch.  Both take numpy arrays or CUDA tensors, return CUDA
tensors and do not wait for the device.  `video_keypoints` is the back half of gen_video_kpts(gen_output=True) on a
chunk of decoded frames.  The kernels are csrc/keypoints2d.cuh; every formula is in DESIGN.md §8.6.

`track_records` and `record_inverse` compute the box geometry on the device from DeviceSort.update_chunk's tracks:
select_tracks, round(v, 2), box_to_center_scale and get_affine_transform with OpenCV's own 6 x 6 LU restated in its
order, equal to the host functions with cv2 bit for bit (csrc/records.cuh, DESIGN.md §8.9).  `video_keypoints` takes
those tracks directly, and then makes one synchronisation per chunk: the copy of the record count and status.

For per-frame track lists the box geometry (box_to_center_scale, get_affine_transform) runs on the host, as do the
drop-ins; it follows the reference's float32 / float64 steps.  The matrices themselves come from
cv2.getAffineTransform when cv2 is importable, which makes the crops and keypoints equal to the reference's bit for
bit.  Without cv2 a closed form in double gives matrices within a few ulps of OpenCV's; a crop warped with them can
then differ from the reference's in a few pixels by one grey level, where the fixed-point warp rounds an exact half.

Refused before any launch (GastError): a box whose width and height are both non-positive (its triangle is
singular), a non-finite box or matrix, a frame side above 32767 (OpenCV keeps source coordinates as int16), a crop
side above 32767, heatmaps of more than 32 joints or with a side above 256, non-float32 heatmaps, a frame index out of
range, and in `video_keypoints` a frame with between 2 and num_person - 1 tracks (the reference's reshape raises).
With DeviceSort's tracks these are found on the device and raised at the call's one copy, with the same messages.
"""
import numpy as np
import torch

from .engine import GastError, _launch, _p

IMAGE_SIZE = (288, 384)          # w48_384x288: MODEL.IMAGE_SIZE (w, h)
PIXEL_STD = 200
RGB_INPUT, NET_ORDER = 1, 2      # gast_person_crops flags
MAX_SIDE = 32767
MAX_HEATMAP, MAX_J = 256, 32

try:
    import cv2 as _cv2
except ImportError:              # the closed form below; see the module docstring
    _cv2 = None


# ------------------------------------------------------------------------------------------------
# box geometry on the host
# ------------------------------------------------------------------------------------------------
def box_to_center_scale(box, model_image_width, model_image_height):
    """center (2,) float32 and scale (2,) float32 of box (x1, y1, x2, y2, ...) as utilitys.py:107-136 computes them.
    PreProcess passes (frame height, frame width) as (model_image_width, model_image_height), so the box is padded to
    the frame's H/W aspect, not the crop's; `center_scale` keeps that."""
    x1, y1, x2, y2 = box[:4]
    bw, bh = x2 - x1, y2 - y1
    if not (np.isfinite(float(x1)) and np.isfinite(float(y1)) and np.isfinite(float(x2)) and np.isfinite(float(y2))):
        raise GastError('keypoints2d: box %s is not finite' % (list(box[:4]),))
    if bw <= 0 and bh <= 0:
        raise GastError('keypoints2d: box %s has a non-positive width and height' % (list(box[:4]),))
    center = np.zeros(2, dtype=np.float32)
    center[0] = x1 + bw * 0.5
    center[1] = y1 + bh * 0.5
    aspect = model_image_width * 1.0 / model_image_height
    if bw > aspect * bh:
        bh = bw * 1.0 / aspect
    elif bw < aspect * bh:
        bw = bh * aspect
    scale = np.array([bw * 1.0 / PIXEL_STD, bh * 1.0 / PIXEL_STD], dtype=np.float32)
    if center[0] != -1:
        scale = scale * np.float32(1.25)
    return center, scale


def center_scale(box, frame_h, frame_w):
    """PreProcess's call (utilitys.py:152): the frame's height and width in the model-size slots"""
    return box_to_center_scale(box, frame_h, frame_w)


def triangles(center, scale, output_size):
    """get_affine_transform's float32 triangles (transforms.py:57-89, rot 0, no shift): src in the frame around the
    box, dst in the output of size (w, h)"""
    center = np.asarray(center, dtype=np.float32)
    src_w = (np.asarray(scale, dtype=np.float32) * np.float32(200.0))[0]
    dst_w, dst_h = output_size
    src = np.zeros((3, 2), dtype=np.float32)
    dst = np.zeros((3, 2), dtype=np.float32)
    src[0] = center
    # get_dir's result is float64: the sum is taken in double and stored into float32
    src[1] = center.astype(np.float64) + np.array([0.0, float(src_w * np.float32(-0.5))])
    dst[0] = [dst_w * 0.5, dst_h * 0.5]
    dst[1] = np.array([dst_w * 0.5, dst_h * 0.5]) + np.array([0, dst_w * -0.5], dtype=np.float32)
    for t in (src, dst):                               # get_3rd_point, in float32
        d = t[0] - t[1]
        t[2] = t[1] + np.array([-d[1], d[0]], dtype=np.float32)
    return src, dst


def _affine(src, dst):
    """the 2x3 double matrix taking the three src points to the dst points"""
    if _cv2 is not None:
        return _cv2.getAffineTransform(np.float32(src), np.float32(dst))
    S = np.vstack([np.asarray(src, np.float64).T, np.ones(3)])
    return np.linalg.solve(S.T, np.asarray(dst, np.float64)).T


def affine_pair(center, scale, image_size=IMAGE_SIZE, heatmap_size=None):
    """(forward, inverse) 2x3 float64: forward maps the frame to the crop of image_size (w, h), what
    cv2.warpAffine receives in PreProcess; inverse maps a heatmap of heatmap_size (w, h) back to the frame, what
    transform_preds applies (None when heatmap_size is None).  cv2.getAffineTransform when cv2 is importable (bit for
    bit the reference's), else a closed form in double that is only within a few ulps of it."""
    src, dst = triangles(center, scale, image_size)
    fwd = _affine(src, dst)
    inv = None
    if heatmap_size is not None:
        _, dst_h = triangles(center, scale, heatmap_size)
        inv = _affine(dst_h, src)
    return fwd, inv


def inverse_matrix(center, scale, heatmap_size):
    """get_affine_transform(center, scale, 0, heatmap_size, inv=1)"""
    src, dst = triangles(center, scale, heatmap_size)
    return _affine(dst, src)


# ------------------------------------------------------------------------------------------------
# the two kernels
# ------------------------------------------------------------------------------------------------
def _device(dev):
    return torch.device('cuda', torch.cuda.current_device()) if dev is None else dev


def _on_device(x, dtype, dev, what):
    """x as a contiguous CUDA tensor of dtype on dev: numpy arrays and CPU tensors are uploaded with one asynchronous
    copy, CUDA tensors converted on the device"""
    if isinstance(x, torch.Tensor):
        if x.is_cuda:
            return x.to(device=dev, dtype=dtype).contiguous()
        x = x.numpy()
    a = np.ascontiguousarray(np.asarray(x), dtype=torch.empty(0, dtype=dtype).numpy().dtype)
    out = torch.empty(a.shape, dtype=dtype, device=dev)
    if a.size:
        out.copy_(torch.from_numpy(a), non_blocking=True)
    return out


def _host_matrices(m, what):
    a = np.asarray(m, dtype=np.float64).reshape(-1, 6)
    if not np.all(np.isfinite(a)):
        raise GastError('keypoints2d: %s are not finite' % what)
    return a


def crop_persons(frames, frame_index, forward_mats, size=IMAGE_SIZE, rgb_input=False, net_order=True):
    """PreProcess's crops (n, 3, h, w) float32 on the device: record r is frame frame_index[r] of frames (F, H, W, 3)
    uint8 warped by forward_mats[r] (2x3, what cv2.warpAffine receives) to size (w, h), then ToTensor and Normalize,
    bit for bit.  frames are BGR as cv2 reads them, or RGB (ffmpeg's rgb24) with rgb_input; the planes come in the
    order the net receives (inputs[:, [2, 1, 0]]), or with net_order=False in the reference's (PreProcess's own).
    Numpy or CUDA inputs; host indices and matrices are checked, CUDA ones are used as they are (an index out of
    range crops a black frame)."""
    if isinstance(frames, torch.Tensor) and frames.is_cuda and frames.dtype != torch.uint8:
        raise GastError('keypoints2d: frames must be uint8')
    shape = tuple(frames.shape)
    if len(shape) != 4 or shape[-1] != 3:
        raise GastError('keypoints2d: frames (F, H, W, 3) expected, got %s' % (shape,))
    F, H, W = int(shape[0]), int(shape[1]), int(shape[2])
    if not (0 < H <= MAX_SIDE and 0 < W <= MAX_SIDE):
        raise GastError('keypoints2d: a %d x %d frame (each side 1 .. %d)' % (W, H, MAX_SIDE))
    w, h = int(size[0]), int(size[1])
    if not (0 < w <= MAX_SIDE and 0 < h <= MAX_SIDE):
        raise GastError('keypoints2d: a %d x %d crop (each side 1 .. %d)' % (w, h, MAX_SIDE))
    idx_cuda = isinstance(frame_index, torch.Tensor) and frame_index.is_cuda
    mats_cuda = isinstance(forward_mats, torch.Tensor) and forward_mats.is_cuda
    if not idx_cuda:
        fi = np.asarray(frame_index, dtype=np.int64).reshape(-1)
        if fi.size and (fi.min() < 0 or fi.max() >= F):
            raise GastError('keypoints2d: frame indices outside [0, %d)' % F)
    if not mats_cuda:
        fm = _host_matrices(forward_mats, 'forward matrices')
    dev = frames.device if isinstance(frames, torch.Tensor) and frames.is_cuda else _device(None)
    if idx_cuda:
        idx = frame_index.to(device=dev, dtype=torch.int32).contiguous().view(-1)
    else:
        idx = _on_device(fi, torch.int32, dev, 'frame_index')
    if mats_cuda:
        mats = forward_mats.to(device=dev, dtype=torch.float64).contiguous().view(-1, 6)
    else:
        mats = _on_device(fm, torch.float64, dev, 'forward_mats')
    n = int(idx.shape[0])
    if int(mats.shape[0]) != n:
        raise GastError('keypoints2d: %d frame indices but %d matrices' % (n, int(mats.shape[0])))
    out = torch.empty((n, 3, h, w), dtype=torch.float32, device=dev)
    if n and F:
        fr = _on_device(frames, torch.uint8, dev, 'frames')
        flags = (RGB_INPUT if rgb_input else 0) | (NET_ORDER if net_order else 0)
        _launch(dev, 'gast_person_crops', _p(fr), F, H, W, _p(idx), _p(mats), n, w, h, flags, _p(out))
    return out


def decode_heatmaps(heatmaps, inverse_mats, post_process=True):
    """get_final_preds of heatmaps (n, J, hh, hw) float32 with the inverse (heatmap -> frame) 2x3 matrices
    inverse_mats (n, 2, 3): preds (n, J, 2) and maxvals (n, J, 1) float32 CUDA tensors, bit for bit.  post_process is
    TEST.POST_PROCESS (the quarter-pixel shift towards the higher neighbour)."""
    if isinstance(heatmaps, torch.Tensor) and heatmaps.dtype != torch.float32:
        raise GastError('keypoints2d: heatmaps must be float32, got %s' % heatmaps.dtype)
    if not isinstance(heatmaps, torch.Tensor) and np.asarray(heatmaps).dtype != np.float32:
        raise GastError('keypoints2d: heatmaps must be float32, got %s' % np.asarray(heatmaps).dtype)
    shape = tuple(heatmaps.shape)
    if len(shape) != 4:
        raise GastError('keypoints2d: heatmaps (n, J, hh, hw) expected, got %s' % (shape,))
    n, J, hh, hw = (int(s) for s in shape)
    if not (0 < J <= MAX_J and 0 < hh <= MAX_HEATMAP and 0 < hw <= MAX_HEATMAP):
        raise GastError('keypoints2d: %d joints of %d x %d heatmaps (J <= %d, sides <= %d)'
                        % (J, hw, hh, MAX_J, MAX_HEATMAP))
    mats_cuda = isinstance(inverse_mats, torch.Tensor) and inverse_mats.is_cuda
    if not mats_cuda:
        im = _host_matrices(inverse_mats, 'inverse matrices')
    dev = heatmaps.device if isinstance(heatmaps, torch.Tensor) and heatmaps.is_cuda else _device(None)
    if mats_cuda:
        mats = inverse_mats.to(device=dev, dtype=torch.float64).contiguous().view(-1, 6)
    else:
        mats = _on_device(im, torch.float64, dev, 'inverse_mats')
    if int(mats.shape[0]) != n:
        raise GastError('keypoints2d: %d heatmap records but %d matrices' % (n, int(mats.shape[0])))
    preds = torch.empty((n, J, 2), dtype=torch.float32, device=dev)
    maxvals = torch.empty((n, J, 1), dtype=torch.float32, device=dev)
    if n:
        hm = _on_device(heatmaps, torch.float32, dev, 'heatmaps')
        _launch(dev, 'gast_heatmap_decode', _p(hm), _p(mats), n, J, hh, hw, 1 if post_process else 0, _p(preds),
                _p(maxvals))
    return preds, maxvals


# ------------------------------------------------------------------------------------------------
# gen_video_kpts(gen_output=True) on a chunk of frames
# ------------------------------------------------------------------------------------------------
def select_tracks(track, num_person):
    """the boxes gen_video_kpts keeps of one frame's tracker output (k, >= 4) (gen_kpts.py:214-226): none for k = 0
    (the frame is dropped), the lone track for k = 1, else the last num_person rows reversed; each coordinate
    rounded to 2 decimals.  (num_person', 4) float64, or None for a dropped frame."""
    if track is None:
        return None
    t = np.asarray(track, dtype=np.float64)
    if t.size == 0:
        return None
    if t.ndim != 2 or t.shape[1] < 4:
        raise GastError('keypoints2d: a frame\'s tracks must be (k, 4) or (k, 5), got %s' % (t.shape,))
    k = t.shape[0]
    if k == 1:
        rows = t[:, :4]
    elif k >= num_person:
        rows = t[k - num_person:, :4][::-1]
    else:
        raise GastError('keypoints2d: %d tracks in a frame for num_person = %d (the reference cannot reshape them)'
                        % (k, num_person))
    return np.round(rows, 2)


def video_keypoints(frames, boxes, pose_net, num_person, image_size=IMAGE_SIZE, post_process=True, rgb_input=False):
    """gen_video_kpts(gen_output=True)'s keypoints and scores of a chunk of decoded frames (gen_kpts.py:194-271),
    with the crop and the decode on the device.

    frames (T, H, W, 3) uint8 (BGR as cv2 reads them, RGB with rgb_input), numpy or CUDA; boxes: T per-frame tracker
    outputs (k, 5) or (k, 4) in frame pixels, or None / empty where nothing was detected, or the (rows, counts,
    status) triple tracking.DeviceSort.update_chunk returns for one sequence of T frames; pose_net: a callable
    mapping the crops (n, 3, h, w) float32 on the device, planes in the net's order, to heatmaps (n, 17, hh, hw)
    float32 on the device (HRNet w48_384x288: 96 x 72).  Every box of the chunk is cropped in one launch, the net runs
    once, and the decode is one launch.  With the triple the boxes' geometry is one launch too (track_records), and
    the call's one synchronisation is the copy of its record count and status to the host.

    Returns keypoints (num_person, T', 17, 2) and scores (num_person, T', 17) float32 on the device, T' the frames with
    at least one track; a slot without a track stays zero.  Feeds device.tools.preprocess.h36m_coco_format."""
    num_person = int(num_person)
    if num_person < 1:
        raise GastError('keypoints2d: num_person must be >= 1')
    shape = tuple(frames.shape)
    if len(shape) != 4 or shape[-1] != 3:
        raise GastError('keypoints2d: frames (T, H, W, 3) expected, got %s' % (shape,))
    T, H, W = int(shape[0]), int(shape[1]), int(shape[2])
    if _is_track_triple(boxes):
        rows, counts, status = boxes
        if rows.dim() != 3 or int(rows.shape[0]) != T:
            raise GastError('keypoints2d: %d frames but tracks %s (one sequence of (T, capacity, 5) rows expected)'
                            % (T, tuple(rows.shape)))
        rec = track_records(rows, counts, status, num_person, (W, H), image_size)
        summary = rec.summary.cpu().numpy()                  # the call's one synchronisation
        _raise_records_error(summary, rows, counts, num_person, (W, H))
        n, t_out = int(summary[0, 0]), int(summary[0, 1])
        dev = frames.device if isinstance(frames, torch.Tensor) and frames.is_cuda else _device(None)
        return _keypoints(frames, dev, n, t_out, num_person, rec.frame[:n], rec.forward[:n], rec.slot[:n],
                          lambda size: record_inverse(rec, size)[:n], pose_net, image_size, post_process, rgb_input)
    if len(boxes) != T:
        raise GastError('keypoints2d: %d frames but %d box lists' % (T, len(boxes)))
    frame_idx, slots, centers, scales, fwd = [], [], [], [], []
    t_out = 0
    for t in range(T):
        rows = select_tracks(boxes[t], num_person)
        if rows is None:
            continue
        for p, box in enumerate(rows[:num_person]):
            c, s = center_scale(box, H, W)
            frame_idx.append(t)
            slots.append(t_out * num_person + p)
            centers.append(c)
            scales.append(s)
            fwd.append(affine_pair(c, s, image_size)[0])
        t_out += 1
    n = len(frame_idx)
    dev = frames.device if isinstance(frames, torch.Tensor) and frames.is_cuda else _device(None)
    return _keypoints(frames, dev, n, t_out, num_person, frame_idx, np.stack(fwd) if n else None,
                      np.asarray(slots, dtype=np.int64),
                      lambda size: np.stack([inverse_matrix(c, s, size) for c, s in zip(centers, scales)]),
                      pose_net, image_size, post_process, rgb_input)


def _keypoints(frames, dev, n, t_out, num_person, frame_idx, fwd, slots, inverse, pose_net, image_size, post_process,
               rgb_input):
    """video_keypoints' crop, net, decode and scatter of n records into t_out frames; inverse((hw, hh)) gives the
    records' inverse matrices once the net's heatmap size is known"""
    J = 17
    kpts = torch.zeros((t_out * num_person, J, 2), dtype=torch.float32, device=dev)
    scores = torch.zeros((t_out * num_person, J), dtype=torch.float32, device=dev)
    if n:
        crops = crop_persons(frames, frame_idx, fwd, image_size, rgb_input=rgb_input, net_order=True)
        with torch.no_grad():
            heat = pose_net(crops)
        if not isinstance(heat, torch.Tensor) or not heat.is_cuda or heat.dim() != 4 or \
                int(heat.shape[0]) != n or int(heat.shape[1]) != J:
            raise GastError('keypoints2d: the pose net must return (%d, %d, hh, hw) heatmaps on the device'
                            % (n, J))
        hh, hw = int(heat.shape[2]), int(heat.shape[3])
        preds, maxvals = decode_heatmaps(heat, inverse((hw, hh)), post_process)
        slot = _on_device(slots, torch.int64, dev, 'slots')
        kpts.index_copy_(0, slot, preds)
        scores.index_copy_(0, slot, maxvals.view(-1, J))
    kpts = kpts.view(t_out, num_person, J, 2).transpose(0, 1).contiguous()
    scores = scores.view(t_out, num_person, J).transpose(0, 1).contiguous()
    return kpts, scores


# ------------------------------------------------------------------------------------------------
# SORT's tracks to crop records on the device
# ------------------------------------------------------------------------------------------------
REC_TRACKS, REC_NONFINITE, REC_EMPTY, REC_MATRIX = 0x100, 0x200, 0x400, 0x800    # GAST_REC_ST_*
SORT_BITS = 0xff                                                                 # SORT's own word


class TrackRecords:
    """track_records' outputs on the device, with room for S * K * num_person records; those past `total` are not
    written.  frame (N,) int32: s * K + t; slot (N,) int64: t' * num_person + p, t' the frame's rank among the
    sequence's kept frames; forward (N, 2, 3) float64: the frame -> crop matrix cv2.warpAffine receives;
    center_scale (N, 4) float32 (center and scale are its views); summary (S, 4) int32: each sequence's records, kept
    frames, status word and first offending frame (-1 for none); total (1,) int32: all sequences' records."""

    def __init__(self, frame, slot, forward, center_scale, summary, total):
        self.frame, self.slot, self.forward, self.center_scale = frame, slot, forward, center_scale
        self.summary, self.total = summary, total

    @property
    def center(self):
        return self.center_scale[:, :2]

    @property
    def scale(self):
        return self.center_scale[:, 2:]


def _is_track_triple(boxes):
    return isinstance(boxes, tuple) and len(boxes) == 3 and all(isinstance(b, torch.Tensor) and b.is_cuda
                                                                 for b in boxes)


def track_records(rows, counts, status, num_person, frame_size, image_size=IMAGE_SIZE):
    """The crop records of every box gen_video_kpts keeps (select_tracks, then center_scale and affine_pair's forward
    matrix, bit for bit) from DeviceSort.update_chunk's outputs: rows (K, capacity, 5) / (S, K, capacity, 5) float64,
    counts (K,) / (S, K) int32 and status (S,) int32, for frames of frame_size (W, H) and crops of image_size (w, h).
    One launch; returns a TrackRecords of CUDA tensors without waiting for the device."""
    if not all(isinstance(x, torch.Tensor) and x.is_cuda for x in (rows, counts, status)):
        raise GastError('keypoints2d: rows, counts and status must be CUDA tensors (DeviceSort.update_chunk\'s)')
    if rows.dtype != torch.float64 or counts.dtype != torch.int32 or status.dtype != torch.int32:
        raise GastError('keypoints2d: float64 rows and int32 counts and status expected, got %s, %s, %s'
                        % (rows.dtype, counts.dtype, status.dtype))
    R = rows[None] if rows.dim() == 3 else rows
    N = counts[None] if counts.dim() == 1 else counts
    if R.dim() != 4 or R.shape[-1] != 5 or tuple(N.shape) != tuple(R.shape[:2]) or tuple(status.shape) != (R.shape[0],):
        raise GastError('keypoints2d: rows %s, counts %s and status %s do not match'
                        % (tuple(rows.shape), tuple(counts.shape), tuple(status.shape)))
    S, K, cap = int(R.shape[0]), int(R.shape[1]), int(R.shape[2])
    num_person = int(num_person)
    if num_person < 1:
        raise GastError('keypoints2d: num_person must be >= 1')
    W, H = int(frame_size[0]), int(frame_size[1])
    w, h = int(image_size[0]), int(image_size[1])
    if not (0 < W <= MAX_SIDE and 0 < H <= MAX_SIDE and 0 < w <= MAX_SIDE and 0 < h <= MAX_SIDE):
        raise GastError('keypoints2d: a %d x %d frame or a %d x %d crop (each side 1 .. %d)' % (W, H, w, h, MAX_SIDE))
    dev = rows.device
    n = S * K * num_person
    frame = torch.empty(n, dtype=torch.int32, device=dev)
    slot = torch.empty(n, dtype=torch.int64, device=dev)
    forward = torch.empty((n, 2, 3), dtype=torch.float64, device=dev)
    cs = torch.empty((n, 4), dtype=torch.float32, device=dev)
    summary = torch.empty((S, 4), dtype=torch.int32, device=dev)
    total = torch.zeros(1, dtype=torch.int32, device=dev)
    R, N, st = R.contiguous(), N.to(device=dev).contiguous(), status.to(device=dev).contiguous()
    _launch(dev, 'gast_track_records', _p(R), _p(N), _p(st), S, K, cap, num_person, W, H, w, h, _p(frame), _p(slot),
            _p(forward), _p(cs), _p(summary), _p(total))
    return TrackRecords(frame, slot, forward, cs, summary, total)


def record_inverse(records, heatmap_size):
    """get_affine_transform(center, scale, 0, heatmap_size, inv=1) of every record: (N, 2, 3) float64 on the device,
    inverse_matrix's bits; rows past records.total are not written.  One launch, no synchronisation."""
    hw, hh = int(heatmap_size[0]), int(heatmap_size[1])
    if not (0 < hw <= MAX_SIDE and 0 < hh <= MAX_SIDE):
        raise GastError('keypoints2d: a %d x %d heatmap (each side 1 .. %d)' % (hw, hh, MAX_SIDE))
    cs = records.center_scale
    dev = cs.device
    n = int(cs.shape[0])
    out = torch.empty((n, 2, 3), dtype=torch.float64, device=dev)
    _launch(dev, 'gast_record_inverse', _p(cs), n, _p(records.total), hw, hh, _p(out))
    return out


def _raise_records_error(summary, rows, counts, num_person, frame_size):
    """GastError with the host path's message for the first sequence whose status word is set: tracking's message
    for SORT's bits; for a frame's bits, select_tracks' or center_scale's own, from one copy of that frame's tracks"""
    bad = np.flatnonzero(summary[:, 2])
    if not bad.size:
        return
    s = int(bad[0])
    word, t = int(summary[s, 2]), int(summary[s, 3])
    if word & SORT_BITS:
        from .tracking import status_message
        raise GastError('tracking: sequence %d: %s' % (s, status_message(word & SORT_BITS)))
    if t >= 0:
        R = rows[None] if rows.dim() == 3 else rows
        N = counts[None] if counts.dim() == 1 else counts
        k = int(N[s, t])
        track = R[s, t, :max(0, min(k, int(R.shape[2])))].cpu().numpy()
        sel = select_tracks(track, num_person)
        for box in sel[:num_person] if sel is not None else ():
            center_scale(box, frame_size[1], frame_size[0])
        raise GastError('keypoints2d: sequence %d frame %d: %d tracks (capacity %d)' % (s, t, k, int(R.shape[2])))
    raise GastError('keypoints2d: forward matrices are not finite')
