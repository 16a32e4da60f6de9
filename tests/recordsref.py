"""numpy restatement of csrc/records.cuh: gen_video_kpts' record rule over SORT's rows, round(v, 2),
box_to_center_scale, get_affine_transform's triangles and OpenCV's 6 x 6 LU (getAffineTransform -> solve(DECOMP_LU) ->
LUImpl), vectorised over boxes.  numpy's float64 and float32 element-wise operations round to nearest and are never
fused, so each line is the step the kernel takes with an explicit intrinsic."""
import numpy as np

ST_TRACKS, ST_NONFINITE, ST_EMPTY, ST_MATRIX = 0x100, 0x200, 0x400, 0x800
LU_EPS = 100 * np.finfo(np.float64).eps
f32, f64 = np.float32, np.float64


def rec_count(k, num_person, cap):
    """records of a frame of k tracks; -1 for a count the host path refuses or that cannot be SORT's"""
    if k < -1 or k > cap:
        return -1
    if k <= 0:
        return 0
    if k == 1:
        return 1
    return num_person if k >= num_person else -1


def round2(v):
    """np.round(v, 2) of float64: rint(v * 100) / 100"""
    with np.errstate(over='ignore', invalid='ignore'):
        return np.rint(np.asarray(v, f64) * 100.0) / 100.0


def center_scale(boxes, H, W):
    """box_to_center_scale of rounded boxes (n, 4) float64 with (H, W) in the model-size slots: centers and scales
    (n, 2) float32, and the status bit of each box (0, ST_NONFINITE or ST_EMPTY)"""
    b = np.asarray(boxes, f64).reshape(-1, 4)
    x1, y1, x2, y2 = b.T
    with np.errstate(over='ignore', invalid='ignore'):
        bw, bh = x2 - x1, y2 - y1
        bits = np.where(~np.isfinite(b).all(1), ST_NONFINITE, np.where((bw <= 0) & (bh <= 0), ST_EMPTY, 0))
        c = np.stack([x1 + bw * 0.5, y1 + bh * 0.5], 1).astype(f32)
        aspect = H * 1.0 / W
        wide, tall = bw > aspect * bh, bw < aspect * bh
        bh = np.where(wide, bw * 1.0 / aspect, bh)
        bw = np.where(~wide & tall, bh * aspect, bw)
        s = np.stack([bw * 1.0 / 200, bh * 1.0 / 200], 1).astype(f32)
        s = np.where((c[:, :1] != -1), s * f32(1.25), s)
    return c, s.astype(f32), bits.astype(np.int64)


def triangles(c, s, size):
    """get_affine_transform's float32 triangles of (n,) boxes for an output (w, h): src, dst (n, 3, 2) float32"""
    c = np.asarray(c, f32).reshape(-1, 2)
    s = np.asarray(s, f32).reshape(-1, 2)
    ow, oh = size
    n = c.shape[0]
    src = np.zeros((n, 3, 2), f32)
    dst = np.zeros((n, 3, 2), f32)
    src_w = s[:, 0] * f32(200.0)
    src[:, 0] = c
    src[:, 1, 0] = (c[:, 0].astype(f64) + 0.0).astype(f32)
    src[:, 1, 1] = (c[:, 1].astype(f64) + (src_w * f32(-0.5)).astype(f64)).astype(f32)
    dst[:, 0] = [ow * 0.5, oh * 0.5]
    dst[:, 1, 0] = f32(ow * 0.5 + 0.0)
    dst[:, 1, 1] = f32(oh * 0.5 + f64(f32(ow * -0.5)))
    for t in (src, dst):
        d = t[:, 0] - t[:, 1]
        t[:, 2, 0] = t[:, 1, 0] + -d[:, 1]
        t[:, 2, 1] = t[:, 1, 1] + d[:, 0]
    return src, dst


def affine(src, dst):
    """cv2.getAffineTransform of (n, 3, 2) float32 point triples: (n, 2, 3) float64.  OpenCV's system, LUImpl's
    pivoting (the first row of largest |A[j][i]|), elimination and back-substitution in its order, and a zero matrix
    when a pivot falls below 100 * DBL_EPSILON."""
    src = np.asarray(src, f32).reshape(-1, 3, 2).astype(f64)
    dst = np.asarray(dst, f32).reshape(-1, 3, 2).astype(f64)
    n = src.shape[0]
    A = np.zeros((n, 6, 6))
    b = np.zeros((n, 6))
    for i in range(3):
        A[:, 2 * i, 0], A[:, 2 * i, 1], A[:, 2 * i, 2] = src[:, i, 0], src[:, i, 1], 1.0
        A[:, 2 * i + 1, 3], A[:, 2 * i + 1, 4], A[:, 2 * i + 1, 5] = src[:, i, 0], src[:, i, 1], 1.0
        b[:, 2 * i], b[:, 2 * i + 1] = dst[:, i, 0], dst[:, i, 1]
    singular = np.zeros(n, bool)
    ar = np.arange(n)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        for i in range(6):
            k = np.full(n, i)
            best = np.abs(A[:, i, i])
            for j in range(i + 1, 6):
                take = np.abs(A[:, j, i]) > best
                best = np.where(take, np.abs(A[:, j, i]), best)
                k = np.where(take, j, k)
            singular |= best < LU_EPS
            Ai, Ak = A[ar, i].copy(), A[ar, k].copy()
            A[ar, i], A[ar, k] = Ak, Ai
            bi, bk = b[ar, i].copy(), b[ar, k].copy()
            b[ar, i], b[ar, k] = bk, bi
            d = -1.0 / A[:, i, i]
            for j in range(i + 1, 6):
                alpha = A[:, j, i] * d
                A[:, j, i + 1:] = A[:, j, i + 1:] + alpha[:, None] * A[:, i, i + 1:]
                b[:, j] = b[:, j] + alpha * b[:, i]
        for i in range(5, -1, -1):
            s = b[:, i].copy()
            for c in range(i + 1, 6):
                s = s - A[:, i, c] * b[:, c]
            b[:, i] = s / A[:, i, i]
    b[singular] = 0.0
    return b.reshape(n, 2, 3)


def box_matrices(boxes, H, W, image_size, heatmap_size=None):
    """rounded boxes (n, 4) -> centers, scales, forward (n, 2, 3), inverse (n, 2, 3) or None, status bits (n,)"""
    c, s, bits = center_scale(boxes, H, W)
    src, dst = triangles(c, s, image_size)
    fwd = affine(src, dst)
    inv = None
    if heatmap_size is not None:
        _, dst_h = triangles(c, s, heatmap_size)
        inv = affine(dst_h, src)
    return c, s, fwd, inv, bits


def track_records(rows, counts, status, num_person, frame_size, image_size, heatmap_size=None):
    """gast_track_records of rows (S, K, cap, 5), counts (S, K), status (S,): a dict of the records (frame, slot,
    forward, center, scale, inverse for heatmap_size) and summary (S, 4)"""
    rows = np.asarray(rows, f64)
    S, K, cap = rows.shape[:3]
    W, H = frame_size
    frame, slot, boxes, summary = [], [], [], np.zeros((S, 4), np.int64)
    for s in range(S):
        kept, bits, first, nrec = 0, 0, -1, 0
        for t in range(K):
            k = int(counts[s][t])
            n = rec_count(k, num_person, cap)
            if n < 0:
                bits |= ST_TRACKS
                first = t if first < 0 else first
            if n <= 0:
                continue
            pick = [0] if k == 1 else [k - 1 - p for p in range(n)]
            b = round2(rows[s, t, pick, :4])
            _, _, fb = center_scale(b, H, W)
            if fb.any():
                bits |= int(np.bitwise_or.reduce(fb))
                first = t if first < 0 else first
            for p in range(n):
                frame.append(s * K + t)
                slot.append(kept * num_person + p)
                boxes.append(b[p])
            kept += 1
            nrec += n
        summary[s] = [nrec, kept, bits | int(status[s]), first]
    boxes = np.asarray(boxes, f64).reshape(-1, 4)
    c, sc, fwd, inv, _ = box_matrices(boxes, H, W, image_size, heatmap_size)
    with np.errstate(invalid='ignore'):
        bad = ~np.isfinite(fwd.reshape(-1, 6)).all(1)
    at = 0
    for s in range(S):
        if bad[at:at + summary[s, 0]].any():
            summary[s, 2] |= ST_MATRIX
        at += summary[s, 0]
    return dict(frame=np.asarray(frame, np.int64), slot=np.asarray(slot, np.int64), forward=fwd, center=c, scale=sc,
                inverse=inv, summary=summary)
