"""Numpy restatement of csrc/keypoints2d.cuh (the person crops and the heatmap decode) and of the host box geometry
(DESIGN.md §8.6), plus the integer-formula frames and heatmaps the keypoints2d goldens and tests are made from."""
from fractions import Fraction

import numpy as np

F32 = np.float32
MEAN = np.array([0.485, 0.456, 0.406], dtype=F32)
STD = np.array([0.229, 0.224, 0.225], dtype=F32)


# ------------------------------------------------------------------------------------------------
# inputs from integer formulas
# ------------------------------------------------------------------------------------------------
def _hash(*idx):
    h = np.uint32(2166136261)
    with np.errstate(over='ignore'):
        for k, v in enumerate(idx):
            h = (h ^ (np.asarray(v, dtype=np.uint32) * np.uint32(0x9E3779B1 + 2 * k))) * np.uint32(16777619)
            h = h ^ (h >> np.uint32(13))
    return h


def synth_frames(T, H, W, seed=0):
    """(T, H, W, 3) uint8: a smooth gradient plus hashed noise, so the warp meets every fraction and neighbour"""
    t = np.arange(T, dtype=np.int64)[:, None, None, None]
    y = np.arange(H, dtype=np.int64)[None, :, None, None]
    x = np.arange(W, dtype=np.int64)[None, None, :, None]
    c = np.arange(3, dtype=np.int64)[None, None, None, :]
    noise = (_hash(t + 1000 * seed, y, x, c) % np.uint32(64)).astype(np.int64)
    return ((x * 3 + y * 5 + c * 40 + t * 17 + seed * 11 + noise) % 256).astype(np.uint8)


def synth_heatmaps(n, J, hh, hw, seed=0):
    """(n, J, hh, hw) float32 in (-0.05, 1.2): hashed noise plus one rational bump per map at a hashed place (only
    correctly rounded operations, so every machine makes the same maps)"""
    i = np.arange(n, dtype=np.int64)[:, None, None, None]
    j = np.arange(J, dtype=np.int64)[None, :, None, None]
    y = np.arange(hh, dtype=np.int64)[None, None, :, None]
    x = np.arange(hw, dtype=np.int64)[None, None, None, :]
    base = (_hash(i + 97 * seed, j, y, x) % np.uint32(2001)).astype(np.float64) / 2000.0 * 0.25 - 0.05
    cy = (_hash(i, j, 7 + seed) % np.uint32(hh)).astype(np.int64)
    cx = (_hash(i, j, 11 + seed) % np.uint32(hw)).astype(np.int64)
    bump = 1.0 / (1.0 + ((y - cy) ** 2 + (x - cx) ** 2).astype(np.float64) / 8.0)
    return (base + bump).astype(F32)


def edge_case_heatmaps(hh, hw):
    """(n, 17, hh, hw) float32: peaks on columns and rows 0, 1, w-2, w-1 and inside, ties, an all-negative map, zero
    differences beside the peak, a NaN map, a NaN after the peak, a NaN difference and +-inf"""
    J = 17
    base = synth_heatmaps(2, J, hh, hw, seed=5) * F32(0.1)
    cases = []
    for c in (0, 1, hw // 2, hw - 2, hw - 1):
        for r in (0, 1, hh // 2, hh - 2, hh - 1):
            cases.append((r, c))
    hm = np.repeat(base, 2, axis=0)[:4].copy()
    k = 0
    for n in range(hm.shape[0]):
        for j in range(J):
            m = hm[n, j]
            r, c = cases[k % len(cases)]
            k += 1
            m[r, c] = F32(2.0 + 0.01 * j)
            if j % 4 == 1 and 0 < c < hw - 1:            # a lower right neighbour: shift left
                m[r, c + 1] = F32(1.5)
            if j % 4 == 2 and 0 < r < hh - 1:            # equal vertical neighbours: zero difference
                m[r - 1, c] = m[r + 1, c] = F32(0.7)
    m = hm[0]
    m[0] = F32(-1.0)                                      # all-negative, ties everywhere: index 0, masked
    m[1] = F32(0.5)                                       # ties everywhere: index 0
    m[2][3, 4] = m[2][6, 9] = F32(3.0)                    # two equal peaks: the first wins
    m[3][:] = np.nan                                      # a NaN map
    m[4][5, 5] = F32(4.0)                                 # a NaN after the peak wins over it
    m[4][hh - 3, hw - 3] = np.nan
    m[5][hh // 2, hw // 2] = F32(4.0)                     # -inf - -inf: a NaN difference, a NaN coordinate
    m[5][hh // 2 - 1, hw // 2] = m[5][hh // 2 + 1, hw // 2] = -np.inf
    m[6][hh // 2, hw // 2] = np.inf                       # inf peak, inf neighbour difference
    m[6][hh // 2 + 1, hw // 2] = np.inf
    m[7][:] = -np.inf
    m[8][:] = F32(-0.25)
    m[8][hh - 2, hw - 2] = F32(-0.1)                      # a negative peak: masked to 0
    m[9][:] = F32(0.0)
    m[9][2, 2] = F32(1e-30)
    return hm


# ------------------------------------------------------------------------------------------------
# host geometry (utilitys.py box_to_center_scale, transforms.py get_affine_transform)
# ------------------------------------------------------------------------------------------------
def center_scale(box, frame_h, frame_w):
    """box_to_center_scale(box, frame_h, frame_w): the aspect is the frame's H/W"""
    x1, y1, x2, y2 = box[:4]
    bw, bh = x2 - x1, y2 - y1
    center = np.zeros(2, F32)
    center[0] = x1 + bw * 0.5
    center[1] = y1 + bh * 0.5
    aspect = frame_h * 1.0 / frame_w
    if bw > aspect * bh:
        bh = bw * 1.0 / aspect
    elif bw < aspect * bh:
        bw = bh * aspect
    scale = np.array([bw / 200.0, bh / 200.0], F32)
    if center[0] != -1:
        scale = scale * F32(1.25)
    return center, scale


def triangles(center, scale, size):
    src_w = scale[0] * F32(200.0)
    w, h = size
    src = np.zeros((3, 2), F32)
    dst = np.zeros((3, 2), F32)
    src[0] = center
    src[1] = [float(center[0]) + 0.0, float(center[1]) - 0.5 * float(src_w)]
    dst[0] = [w * 0.5, h * 0.5]
    dst[1] = [w * 0.5, h * 0.5 - w * 0.5]
    for t in (src, dst):
        d = t[0] - t[1]
        t[2] = t[1] + np.array([-d[1], d[0]], F32)
    return src, dst


# ------------------------------------------------------------------------------------------------
# gast_person_crops
# ------------------------------------------------------------------------------------------------
def invert(M):
    """warpAffine's inverse of the forward 2x3 matrix (the fixed-point path's M)"""
    M = np.asarray(M, np.float64).reshape(6).copy()
    D = M[0] * M[4] - M[1] * M[3]
    D = 1.0 / D if D != 0 else 0.0
    A11, A22 = M[4] * D, M[0] * D
    M[0] = A11
    M[1] *= -D
    M[3] *= -D
    M[4] = A22
    b1 = -M[0] * M[2] - M[1] * M[5]
    b2 = -M[3] * M[2] - M[4] * M[5]
    M[2], M[5] = b1, b2
    return M


def warp(img, M, w, h):
    """cv2.warpAffine(img, M, (w, h), flags=INTER_LINEAR), constant 0 border, by OpenCV's fixed-point path"""
    m = invert(M)
    xs, ys = np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64)
    ad = np.rint(m[0] * xs * 1024).astype(np.int64)
    bd = np.rint(m[3] * xs * 1024).astype(np.int64)
    X0 = np.rint((m[1] * ys + m[2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((m[4] * ys + m[5]) * 1024).astype(np.int64) + 16
    X = (X0[:, None] + ad[None, :]) >> 5
    Y = (Y0[:, None] + bd[None, :]) >> 5
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    fx, fy = X & 31, Y & 31
    H, W = img.shape[:2]

    def px(yy, xx):
        ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        v = img[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)].astype(np.int64)
        return np.where(ok[..., None], v, 0)
    w00 = ((32 - fx) * (32 - fy) * 32)[..., None]
    w01 = (fx * (32 - fy) * 32)[..., None]
    w10 = ((32 - fx) * fy * 32)[..., None]
    w11 = (fx * fy * 32)[..., None]
    v = px(sy, sx) * w00 + px(sy, sx + 1) * w01 + px(sy + 1, sx) * w10 + px(sy + 1, sx + 1) * w11
    return np.clip((v + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def normalize(u8, rgb_input=False, net_order=True):
    """ToTensor + Normalize of an (h, w, 3) warp: (3, h, w) float32, statistics c on BGR plane c"""
    bgr = u8[..., ::-1] if rgb_input else u8
    v = np.ascontiguousarray(bgr.transpose(2, 0, 1)).astype(F32) / F32(255)
    out = (v - MEAN[:, None, None]) / STD[:, None, None]
    return out[::-1].copy() if net_order else out


def crop(frame, M, size, rgb_input=False, net_order=True):
    return normalize(warp(frame, M, size[0], size[1]), rgb_input, net_order)


# ------------------------------------------------------------------------------------------------
# gast_heatmap_decode
# ------------------------------------------------------------------------------------------------
def _fma(a, b, c):
    return float(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _apply(m, x, y):
    """np.dot(m, [x, y, 1]) as numpy's BLAS evaluates it: fma(m0, x, m1 * y) + m2, stored into float32"""
    x, y = float(x), float(y)
    if np.isnan(x) or np.isnan(y):
        return F32(np.nan)
    return F32(_fma(m[0], x, float(m[1]) * y) + float(m[2]))


def decode(hm, inv, post_process=True):
    """get_final_preds of hm (n, J, hh, hw) float32 with inverse matrices (n, 2, 3): preds (n, J, 2), maxvals (n, J, 1)"""
    n, J, hh, hw = hm.shape
    inv = np.asarray(inv, np.float64).reshape(n, 2, 3)
    preds = np.zeros((n, J, 2), F32)
    maxvals = np.zeros((n, J, 1), F32)
    flat = hm.reshape(n, J, -1)
    for i in range(n):
        for j in range(J):
            idx = int(np.argmax(flat[i, j]))
            mv = flat[i, j, idx]
            mask = F32(1) if mv > 0 else F32(0)
            x = F32(idx % hw) * mask
            y = F32(np.floor(F32(idx) / F32(hw))) * mask
            if post_process:
                px, py = int(x), int(y)
                if 1 < px < hw - 1 and 1 < py < hh - 1:
                    m = hm[i, j]
                    with np.errstate(invalid='ignore'):
                        x = F32(x + np.sign(F32(m[py, px + 1] - m[py, px - 1])) * F32(0.25))
                        y = F32(y + np.sign(F32(m[py + 1, px] - m[py - 1, px])) * F32(0.25))
            preds[i, j, 0] = _apply(inv[i, 0], x, y)
            preds[i, j, 1] = _apply(inv[i, 1], x, y)
            maxvals[i, j, 0] = mv
    return preds, maxvals
