"""numpy restatement of the person detector's letterbox and post-processing (csrc/detect.cuh, DESIGN.md §8.7):
gast_letterbox (preprocess.prep_image: letterbox_image's cv2.resize(INTER_CUBIC) into a 128 canvas, BGR -> RGB,
/255) and gast_person_detections (util.write_results(det_hm=True) plus yolo_human_det's rescale, clamp and round).
Every step is float32 or an exact integer step, in the kernels' order; the tests compare bit for bit.

Frames and predictions are made by integer formulas here, so the goldens need not store them."""
import numpy as np

f32 = np.float32
COEF_SCALE = 2048                   # INTER_RESIZE_COEF_SCALE: 11-bit short coefficients
SIMD_STEP = 8                       # the vertical pass's 128-bit float path covers 8 interleaved values per step
STRIDES = (32, 16, 8)
ATTRS = 85


# ------------------------------------------------------------------------------------------------
# inputs from integer formulas
# ------------------------------------------------------------------------------------------------
def synth_frames(F, H, W, seed=0):
    """(F, H, W, 3) uint8 BGR: gradients, a checkerboard and a per-seed hash, so every tap of the cubic kernel sees
    structure and the 0 / 255 saturation is reached"""
    y = np.arange(H, dtype=np.int64)[:, None]
    x = np.arange(W, dtype=np.int64)[None, :]
    out = np.empty((F, H, W, 3), np.uint8)
    for f in range(F):
        s = seed * 7 + f
        h = (x * 2654435761 + y * 40503 + s * 97) & 0xffff
        out[f, :, :, 0] = ((x * 255) // max(W - 1, 1) + s * 13) % 256
        out[f, :, :, 1] = np.where(((x // 9) + (y // 7) + s) % 2 == 0, 250, 5)
        out[f, :, :, 2] = (h >> 8) % 256
    return out


def num_predictions(D):
    """N = 3 * sum((D / s)^2) over the three YOLO scales"""
    return 3 * sum((D // s) ** 2 for s in STRIDES)


# ------------------------------------------------------------------------------------------------
# letterbox (gast_letterbox)
# ------------------------------------------------------------------------------------------------
def letterbox_geometry(W, H, D):
    """(new_w, new_h, off_x, off_y): letterbox_image's double expression and paste offsets"""
    new_w = int(W * min(D / W, D / H))
    new_h = int(H * min(D / W, D / H))
    return new_w, new_h, (D - new_w) // 2, (D - new_h) // 2


def cubic_coeffs(fx):
    """interpolateCubic (A = -0.75) in float32, the last coefficient 1 - the other three, as 11-bit shorts"""
    A = f32(-0.75)
    fx = np.asarray(fx, f32)
    x1 = fx + f32(1)
    c0 = ((A * x1 - f32(-3.75)) * x1 + f32(-6)) * x1 - f32(-3)
    c1 = (f32(1.25) * fx - f32(2.25)) * fx * fx + f32(1)
    om = f32(1) - fx
    c2 = (f32(1.25) * om - f32(2.25)) * om * om + f32(1)
    c3 = f32(1) - c0 - c1 - c2
    c = np.stack([c0, c1, c2, c3], -1).astype(f32)
    return np.clip(np.rint(c * f32(COEF_SCALE)), -32768, 32767).astype(np.int64)


def resize_axis(src, dst):
    """source indices (dst, 4), clamped to the edge, and short coefficients (dst, 4) of one axis"""
    scale = 1.0 / (float(dst) / src)
    d = np.arange(dst, dtype=np.float64)
    f = ((d + 0.5) * scale - 0.5).astype(f32)
    s = np.floor(f).astype(np.int64)
    f = (f - s.astype(f32)).astype(f32)
    idx = np.clip(s[:, None] + np.arange(-1, 3)[None, :], 0, src - 1)
    return idx, cubic_coeffs(f)


def resize_cubic(img, new_w, new_h):
    """cv2.resize(img, (new_w, new_h), interpolation=INTER_CUBIC) of a (H, W, 3) uint8 image, OpenCV's own path: the
    horizontal pass in int32; the vertical pass in float32 (unfused multiply-adds, round half to even) for the first
    8 * floor(3 new_w / 8) interleaved values of each row and FixedPtCast<int, uchar, 22> for the rest"""
    H, W = img.shape[:2]
    xi, xw = resize_axis(W, new_w)
    yi, yw = resize_axis(H, new_h)
    a = img.astype(np.int64)
    h = (a[:, xi, :] * xw[None, :, :, None]).sum(2).reshape(H, -1)          # (H, 3 new_w)
    S = np.stack([h[yi[:, k]] for k in range(4)], 1)                        # (new_h, 4, 3 new_w)
    fixed = np.clip((np.einsum('ykx,yk->yx', S, yw) + (1 << 21)) >> 22, 0, 255)
    b = yw.astype(f32) * f32(1.0 / (COEF_SCALE * COEF_SCALE))
    Sf = S.astype(f32)
    t = Sf[:, 3] * b[:, 3:4]
    for k in (2, 1, 0):
        t = (Sf[:, k] * b[:, k:k + 1]).astype(f32) + t
    flt = np.clip(np.rint(t), 0, 255)
    width = 3 * new_w
    nvec = (width // SIMD_STEP) * SIMD_STEP
    out = fixed.copy()
    out[:, :nvec] = flt[:, :nvec]
    return out.astype(np.uint8).reshape(new_h, new_w, 3)


def letterbox_u8(frame, D):
    """letterbox_image: (D, D, 3) canvas of 128 with the resized frame pasted, channels as the frame's"""
    H, W = frame.shape[:2]
    nw, nh, ox, oy = letterbox_geometry(W, H, D)
    canvas = np.full((D, D, 3), 128, np.uint8)
    canvas[oy:oy + nh, ox:ox + nw] = resize_cubic(frame, nw, nh)
    return canvas


def to_planes(canvas_u8, rgb_input=False):
    """img[:, :, ::-1].transpose(2, 0, 1) / 255 in float32 (a correctly rounded division)"""
    c = canvas_u8 if rgb_input else canvas_u8[:, :, ::-1]
    return (c.transpose(2, 0, 1).astype(f32) / f32(255)).astype(f32)


def letterbox(frames, D, rgb_input=False):
    """(F, 3, D, D) float32: prep_image of every frame (RGB input: the frames' channels reversed)"""
    out = []
    for fr in frames:
        bgr = fr[:, :, ::-1] if rgb_input else fr
        out.append(to_planes(letterbox_u8(np.ascontiguousarray(bgr), D)))
    return np.stack(out)


# ------------------------------------------------------------------------------------------------
# post-processing (gast_person_detections)
# ------------------------------------------------------------------------------------------------
def _tmax(a, b):
    return f32(np.nan) if (a != a or b != b) else (b if a < b else a)


def _tmin(a, b):
    return f32(np.nan) if (a != a or b != b) else (b if b < a else a)


def iou(b1, b2):
    """bbox_iou with its +1 areas, float32, NaN propagating through torch.max / torch.min"""
    with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
        ix1, iy1 = _tmax(b1[0], b2[0]), _tmax(b1[1], b2[1])
        ix2, iy2 = _tmin(b1[2], b2[2]), _tmin(b1[3], b2[3])
        inter = _tmax(f32(ix2 - ix1) + f32(1), f32(0)) * _tmax(f32(iy2 - iy1) + f32(1), f32(0))
        a1 = f32(f32(b1[2] - b1[0]) + f32(1)) * f32(f32(b1[3] - b1[1]) + f32(1))
        a2 = f32(f32(b2[2] - b2[0]) + f32(1)) * f32(f32(b2[3] - b2[1]) + f32(1))
        return f32(f32(inter) / f32(f32(a1 + a2) - f32(inter)))


def candidates(pred, confidence):
    """the rows of one frame's (N, 85) predictions write_results keeps before the sort: [(row, box (4,), obj,
    max_conf)] in row order, and the number of rows that reach the person filter's count (obj != 0 and argmax 0)"""
    conf = f32(confidence)
    out, persons = [], 0
    with np.errstate(invalid='ignore', over='ignore'):
        for r in range(pred.shape[0]):
            row = pred[r]
            m = f32(1) if row[4] > conf else f32(0)
            obj = f32(row[4] * m)
            if obj == 0:
                continue
            s = (row[5:] * m).astype(f32)
            nan = np.isnan(s)
            if nan.any():
                if not nan[0]:
                    continue
            elif s[0] < s[1:].max():
                continue
            persons += 1
            if s[0] == 0:
                continue
            x, y, w, h = (f32(v * m) for v in row[:4])
            out.append((r, np.array([x - w / f32(2), y - h / f32(2), x + w / f32(2), y + h / f32(2)], f32), obj, s[0]))
    return out, persons


def sort_key(c):
    """objectness descending, NaN first; ties keep the lower prediction index first (the device's rule)"""
    obj = c[2]
    return (0 if np.isnan(obj) else 1, -float(obj), c[0])


def nms(cands, nms_thresh):
    """write_results' greedy loop on the sorted candidates: a later row is multiplied by 0 unless iou < nms_thresh,
    then dropped if its objectness is 0 (a non-finite objectness stays, NaN, with its box zeroed)"""
    thr = f32(nms_thresh)
    rows = [[c[0], c[1].copy(), c[2], c[3]] for c in sorted(cands, key=sort_key)]
    i = 0
    with np.errstate(invalid='ignore', over='ignore'):
        while i < len(rows):
            keep = [rows[k] for k in range(i + 1)]
            for k in range(i + 1, len(rows)):
                if not (iou(rows[i][1], rows[k][1]) < thr):
                    rows[k][1] = (rows[k][1] * f32(0)).astype(f32)
                    rows[k][2] = f32(rows[k][2] * f32(0))
                    rows[k][3] = f32(rows[k][3] * f32(0))
                    if rows[k][2] == 0:
                        continue
                keep.append(rows[k])
            rows = keep
            i += 1
    return rows


def scale_factor(D, W, H):
    """torch.min(inp_dim / img_dim, 1): the python int over a float32 tensor is its reciprocal times D"""
    return min(f32(f32(1) / f32(W)) * f32(D), f32(f32(1) / f32(H)) * f32(D))


def round2(v):
    """round(np.float32, 2): rint(v * 100) / 100 in float32"""
    v = np.asarray(v, f32)
    with np.errstate(invalid='ignore', over='ignore'):
        return (np.rint(v * f32(100)) / f32(100)).astype(f32)


def rescale(box, D, W, H):
    """yolo_human_det's rescale, clamp and round of one (4,) float32 box"""
    sf = scale_factor(D, W, H)
    with np.errstate(invalid='ignore', over='ignore'):
        px = f32(f32(f32(D) - f32(sf * f32(W))) / f32(2))
        py = f32(f32(f32(D) - f32(sf * f32(H))) / f32(2))
        b = np.array([box[0] - px, box[1] - py, box[2] - px, box[3] - py], f32) / sf
        out = []
        for k, lim in enumerate((W, H, W, H)):
            v = b[k]
            v = v if not (v < 0) else f32(0)                     # std::max(v, 0), NaN kept
            v = f32(lim) if f32(lim) < v else v                    # std::min(v, lim)
            out.append(v)
    return round2(np.array(out, f32))


def person_boxes(pred, frame_sizes, D, confidence=0.7, nms_thresh=0.4, max_det=100, raw=False):
    """(boxes (F, K, 4), scores (F, K), counts (F,), max_conf (F, K), persons (F,)): every frame's survivors in
    order, rescaled to frame pixels and rounded (or left as write_results' corners with raw), zero past the count"""
    pred = np.asarray(pred, f32)
    F = pred.shape[0]
    boxes = np.zeros((F, max_det, 4), f32)
    scores = np.zeros((F, max_det), f32)
    mconf = np.zeros((F, max_det), f32)
    counts = np.zeros(F, np.int32)
    persons = np.zeros(F, np.int32)
    for f in range(F):
        cands, persons[f] = candidates(pred[f], confidence)
        rows = nms(cands, nms_thresh)
        counts[f] = len(rows)
        W, H = (int(v) for v in frame_sizes[f])
        for k, r in enumerate(rows[:max_det]):
            boxes[f, k] = r[1] if raw else rescale(r[1], D, W, H)
            scores[f, k] = r[2]
            mconf[f, k] = r[3]
    return boxes, scores, counts, mconf, persons


# ------------------------------------------------------------------------------------------------
# prediction sets for the goldens and tests
# ------------------------------------------------------------------------------------------------
def uniform(seed, n, lo=0.0, hi=1.0):
    """n float64 values in [lo, hi) from an integer hash of (seed, index): the same on every numpy"""
    i = np.arange(n, dtype=np.uint64)
    h = (i * np.uint64(2654435761) + np.uint64(seed) * np.uint64(40503) + np.uint64(12345)) & np.uint64(0xffffffff)
    h = ((h ^ (h >> np.uint64(15))) * np.uint64(2246822519)) & np.uint64(0xffffffff)
    h = ((h ^ (h >> np.uint64(13))) * np.uint64(3266489917)) & np.uint64(0xffffffff)
    h = h ^ (h >> np.uint64(16))
    return lo + (hi - lo) * (h.astype(np.float64) / 4294967296.0)


def background(D, seed):
    """(N, 85) float32 below any threshold: objectness in (0, 0.3), centres on the grid, class scores in (0, 0.5)"""
    N = num_predictions(D)
    p = np.empty((N, ATTRS), f32)
    p[:, 0] = uniform(seed * 11 + 1, N, 0, D)
    p[:, 1] = uniform(seed * 11 + 2, N, 0, D)
    p[:, 2] = uniform(seed * 11 + 3, N, 4, D / 3)
    p[:, 3] = uniform(seed * 11 + 4, N, 4, D / 2)
    p[:, 4] = uniform(seed * 11 + 5, N, 0.0, 0.3)
    p[:, 5:] = uniform(seed * 11 + 6, N * 80, 0.0, 0.5).reshape(N, 80)
    return p


def put(p, row, cx, cy, w, h, obj, cls=0, score=0.9):
    """a detection at row: centre, size, objectness and its best class"""
    p[row, :4] = (cx, cy, w, h)
    p[row, 4] = obj
    p[row, 5:] = f32(0.05)
    p[row, 5 + cls] = score
    return p


def prediction_sets():
    """name -> (D, (N, 85) float32, nms_thresh, frame (W, H)): none passing, candidates but no person, a single
    survivor, overlaps at IoU just either side of 0.4, boxes partly outside the frame, NaN objectness, several D"""
    sets = {}
    D = 416
    N = num_predictions(D)
    sets['none'] = (D, background(D, 1), 0.4, (1920, 1080))
    p = background(D, 2)
    put(p, 100, 200, 200, 50, 120, 0.95, cls=2)
    put(p, 2000, 100, 300, 40, 80, 0.85, cls=15)
    sets['no_person'] = (D, p, 0.4, (1920, 1080))
    p = background(D, 3)
    put(p, 5000, 180.3, 210.7, 60.2, 150.9, 0.93)
    sets['single'] = (D, p, 0.4, (1920, 1080))
    # two pairs of equal boxes, shifted so the IoU is just under and just over 0.4
    p = background(D, 4)
    put(p, 10, 100.0, 200.0, 100.0, 100.0, 0.99)
    put(p, 11, 100.0 + 43.0, 200.0, 100.0, 100.0, 0.98)       # iou = 58*101/(2*10201 - 58*101) = 0.4032 -> dropped
    put(p, 3000, 300.0, 200.0, 100.0, 100.0, 0.97)
    put(p, 3001, 300.0 + 44.0, 200.0, 100.0, 100.0, 0.96)     # iou = 57*101/(2*10201 - 57*101) = 0.3931 -> kept
    put(p, 7000, 300.0 + 44.0, 205.0, 90.0, 90.0, 0.80, cls=3)    # not a person
    sets['iou_edge'] = (D, p, 0.4, (1920, 1080))
    p = background(D, 5)
    put(p, 20, 5.0, 150.0, 60.0, 200.0, 0.91)                 # left edge, above the padding
    put(p, 9000, 410.0, 300.0, 50.0, 400.0, 0.88)             # right and bottom edge
    put(p, 600, 200.0, 70.0, 80.0, 100.0, 0.87)               # into the top padding band
    put(p, 8000, 250.0, 350.0, 120.0, 100.0, 0.86)            # into the bottom padding band
    sets['clamp'] = (D, p, 0.4, (1920, 1080))
    p = background(D, 6)
    p[30, 4] = np.nan                                          # NaN objectness, finite class scores: dropped
    put(p, 31, 100.0, 100.0, 50.0, 90.0, np.nan)
    p[31, 5] = np.nan                                          # NaN objectness and class 0: kept, box zeroed
    put(p, 700, 120.0, 110.0, 50.0, 90.0, 0.95)
    put(p, 701, 122.0, 112.0, 52.0, 88.0, 0.94)                # suppressed by 700
    put(p, 4000, 300.0, 250.0, 70.0, 140.0, 0.9)
    p[4001, 4] = 0.99
    p[4001, 5:] = f32(0.1)
    p[4001, 7] = np.nan                                        # a NaN class score wins the argmax: not a person
    sets['nan'] = (D, p, 0.4, (1280, 720))
    for D, (W, H), nt in ((160, (641, 481), 0.45), (320, (1080, 1920), 0.4), (608, (320, 240), 0.3)):
        p = background(D, D)
        N = num_predictions(D)
        rows = (np.arange(24) * 7919 + D) % N
        objs = np.linspace(0.72, 0.99, 24).astype(f32)[(np.arange(24) * 7) % 24]
        u = uniform(D + 1, 4 * 24).reshape(24, 4)
        for k, r in enumerate(rows):
            put(p, r, u[k, 0] * D, u[k, 1] * D, 10 + u[k, 2] * D / 3, 20 + u[k, 3] * D / 2, objs[k],
                cls=0 if k % 5 else 1 + k)
        sets['d%d' % D] = (D, p, nt, (W, H))
    return sets


def many_candidates(D, n, seed, ties=False):
    """(N, 85) with n person candidates scattered over the image, about two dominant ones; with ties, objectness on a
    coarse grid including exact 1.0 (a saturated sigmoid)"""
    p = background(D, seed)
    N = num_predictions(D)
    rows = np.unique((np.arange(n, dtype=np.int64) * 7919 + seed * 31) % N)
    u = uniform(seed + 1000, 5 * len(rows)).reshape(-1, 5)
    for k, r in enumerate(rows):
        if ties:
            obj = [1.0, 0.9, 0.9, 0.8][k % 4]
        else:
            obj = 0.99 - 0.05 * u[k, 0] if k < 2 else 0.71 + 0.2 * u[k, 0]
        cx, cy = (u[k, 1] * D, u[k, 2] * D) if k >= 2 else (120 + 180 * k, 200)
        put(p, r, cx, cy, 20 + 100 * u[k, 3], 40 + 160 * u[k, 4], obj)
    return p
