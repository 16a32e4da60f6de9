"""numpy float32 restatement of the animation rasteriser (csrc/render.cuh, DESIGN.md §8.5) and of render_frames' frame
selection (gast_b200/render.py Scene, after vis_h36m.py:121-155).  Every operation is one correctly rounded float32
operation in the kernel's order, so the device frames must equal these bit for bit."""
import numpy as np

f32 = np.float32
SHARED_PANEL, FOLLOW_ROOT, BONES_2D = 1, 2, 4
PINK = (255., 192., 203.)


def downsample(x, factor):
    """downsample_tensor: float32 as a sequential float32 sum over each group then one division; uint8 as numpy's
    float64 mean of the integers, truncated by astype('uint8')"""
    n = x.shape[0] // factor
    g = x[:n * factor].reshape((n, factor) + x.shape[1:])
    if x.dtype == np.uint8:
        return (g.astype(np.int64).sum(1).astype(np.float64) / factor).astype(np.uint8)
    acc = g[:, 0].astype(f32)
    for k in range(1, factor):
        acc = acc + g[:, k]
    return acc / f32(factor)


def reference_downsample(x, factor):
    """the reference's downsample_tensor expression (vis_h36m.py:53-55), for the CPU test to hold downsample to"""
    length = x.shape[0] // factor * factor
    return np.mean(x[:length].reshape(-1, factor, *x.shape[1:]), axis=1)


def scene(keypoints, poses, input_frames=None, limit=-1, factor=1, skip=0):
    """render_frames' inputs after the frame selection: (kp (n,M,J,2), poses (P,n,J,3), video or None, n_frames)"""
    kp = np.asarray(keypoints, dtype=f32)
    if kp.ndim == 3:
        kp = kp[:, None]
    ps = [np.asarray(p, dtype=f32) for p in poses]
    vid = None
    if input_frames is not None:
        vid = np.asarray(input_frames, dtype=np.uint8)
        vid = vid[skip:] if limit == -1 else vid[skip:max(limit, skip)]
        kp, ps = kp[skip:], [p[skip:] for p in ps]
    n = min([len(kp)] + [len(p) for p in ps] + ([len(vid)] if vid is not None else []))
    kp, ps = kp[:n], [p[:n] for p in ps]
    vid = vid[:n] if vid is not None else None
    if factor > 1:
        kp, ps = downsample(kp, factor), [downsample(p, factor) for p in ps]
        vid = downsample(vid, factor) if vid is not None else None
    n //= factor
    return kp, np.stack(ps), vid, (n if limit < 1 else min(limit, n))


def _clamp01(x):
    return np.fmin(np.fmax(x, f32(0)), f32(1))


def _lerp(c, target, cov):
    return c + cov * (f32(target) - c)


def _seg(X, Y, a, b):
    """distance from the pixel centres to the segment a -> b, and the nearest point's parameter (seg_dist)"""
    wx, wy = X - a[0], Y - a[1]
    dx, dy = b[0] - a[0], b[1] - a[1]
    l2 = dx * dx + dy * dy
    if l2 > 0:
        t = _clamp01((wx * dx + wy * dy) / l2)
    else:
        t = np.zeros_like(wx)
    ex, ey = wx - t * dx, wy - t * dy
    return np.sqrt(ex * ex + ey * ey), t


def _input_panel(X, Y, pts, image, Hin, Win, M, J, parents, right, n_bones, flags, geo):
    u = (X - geo[13]) / geo[12] - f32(0.5)
    v = (Y - geo[14]) / geo[12] - f32(0.5)
    inside = (u >= f32(-0.5)) & (u < f32(Win) - f32(0.5)) & (v >= f32(-0.5)) & (v < f32(Hin) - f32(0.5))
    c = np.full(u.shape + (3,), 255., dtype=f32)
    if image is None:
        c[inside] = 0.
    else:
        x0, y0 = np.floor(u), np.floor(v)
        fx, fy = u - x0, v - y0
        gx, gy = f32(1) - fx, f32(1) - fy
        xi, yi = x0.astype(np.int64), y0.astype(np.int64)
        xa, xb = np.clip(xi, 0, Win - 1), np.clip(xi + 1, 0, Win - 1)
        ya, yb = np.clip(yi, 0, Hin - 1), np.clip(yi + 1, 0, Hin - 1)
        im = image.astype(f32)
        for ch in range(3):
            top = gx * im[ya, xa, ch] + fx * im[ya, xb, ch]
            bot = gx * im[yb, xa, ch] + fx * im[yb, xb, ch]
            c[..., ch] = np.where(inside, gy * top + fy * bot, c[..., ch])
    if flags & BONES_2D:
        cov = np.zeros(u.shape, dtype=f32)
        for m in range(M):
            for j in range(1, n_bones):
                if parents[j] < 0:
                    continue
                d, _ = _seg(X, Y, pts[m * J + j], pts[m * J + parents[j]])
                cov = np.fmax(cov, _clamp01(geo[16] - d))
        for ch in range(3):
            c[..., ch] = np.where(cov > 0, _lerp(c[..., ch], PINK[ch], cov), c[..., ch])
    for i in range(M * J):
        dx, dy = X - pts[i][0], Y - pts[i][1]
        d = np.sqrt(dx * dx + dy * dy)
        co, ci = _clamp01(geo[18] - d), _clamp01(geo[17] - d)
        fill = (255., 0., 0.) if (i % J) in right else (0., 0., 0.)
        for ch in range(3):
            c[..., ch] = np.where(co > 0, _lerp(_lerp(c[..., ch], 255., co), fill[ch], ci), c[..., ch])
    return c


def _pose_panel(X, Y, pts, n_ent, J, parents, colors, n_bones, geo):
    best_z = np.full(X.shape, np.inf, dtype=f32)
    best_cov = np.zeros(X.shape, dtype=f32)
    best_j = np.full(X.shape, -1, dtype=np.int64)
    for e in range(n_ent):
        for j in range(1, n_bones):
            if parents[j] < 0:
                continue
            a, b = pts[e * J + j], pts[e * J + parents[j]]
            d, t = _seg(X, Y, a, b)
            cov = geo[15] - d
            z = a[2] + t * (b[2] - a[2])
            upd = (cov > 0) & (z < best_z)
            best_z = np.where(upd, z, best_z)
            best_cov = np.where(upd, np.fmin(cov, f32(1)), best_cov)
            best_j = np.where(upd, j, best_j)
    c = np.full(X.shape + (3,), 255., dtype=f32)
    col = np.asarray(colors, dtype=f32)[np.maximum(best_j, 0)]
    for ch in range(3):
        c[..., ch] = np.where(best_j >= 0, _lerp(f32(255.), col[..., ch], best_cov), c[..., ch])
    return c


def _project(q, geo, follow_root):
    q = q.astype(f32).copy()
    if follow_root:
        q[:, 0] = q[:, 0] - q[0, 0]
        q[:, 1] = q[:, 1] - q[0, 1]
    r = [((geo[4 * k] * q[:, 0] + geo[4 * k + 1] * q[:, 1]) + geo[4 * k + 2] * q[:, 2]) + geo[4 * k + 3]
         for k in range(3)]
    return np.stack([geo[19] + r[0] / r[2], geo[19] + r[1] / r[2], r[2]], 1)


def render(kp, poses, video, Hin, Win, parents, colors, right, n_bones, S, geo, flags, frames):
    """frames (list of indices) of kp (n,M,J,2), poses (P,n,J,3), video (n,Hin,Win,3) or None -> (F,S,S*(1+panels),3)"""
    geo = np.asarray(geo, dtype=f32)
    M, J = kp.shape[1], kp.shape[2]
    P = poses.shape[0]
    shared = bool(flags & SHARED_PANEL)
    panels = 1 if shared else P
    right = set(int(r) for r in right)
    X, Y = np.meshgrid(np.arange(S, dtype=f32) + f32(0.5), np.arange(S, dtype=f32) + f32(0.5))
    out = np.empty((len(frames), S, S * (1 + panels), 3), dtype=np.uint8)
    for fi, g in enumerate(frames):
        k = kp[g].reshape(M * J, 2).astype(f32)
        pts = np.stack([geo[13] + (k[:, 0] + f32(0.5)) * geo[12], geo[14] + (k[:, 1] + f32(0.5)) * geo[12]], 1)
        cs = [_input_panel(X, Y, pts, None if video is None else video[g], Hin, Win, M, J, parents, right, n_bones,
                           flags, geo)]
        for q in range(panels):
            ents = range(P) if shared else [q]
            pts = np.concatenate([_project(poses[e, g], geo, flags & FOLLOW_ROOT) for e in ents])
            cs.append(_pose_panel(X, Y, pts, len(ents), J, parents, colors, n_bones, geo))
        for q, c in enumerate(cs):
            out[fi, :, q * S:(q + 1) * S] = np.clip(np.rint(c), 0, 255).astype(np.uint8)
    return out
