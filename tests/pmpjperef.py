"""numpy port of p_mpjpe_kernel's per-frame arithmetic (csrc/pipeline.cuh), for the CPU tests of its 3x3 alignment.

Test infrastructure, CPU only.  Frames are batched along the first axis; every step is the kernel's double arithmetic
in the kernel's order (the warp sums become numpy sums, so the last bits differ).  `rotation` is the fixed routine:
U is built by Gram-Schmidt from H v_k, so it is orthonormal whatever the rank of H.  `rotation_pre_fix` is the routine
it replaced (U[:, k] = H v_k / sqrt(lambda_k), a cross product only below s2 <= 1e-9 s0), kept to show which frames it
got wrong.
"""
import numpy as np

NOISE = 1e-12      # PM_NOISE: |H v| below this times s0 is rounding noise


def jacobi_eig3(a):
    """jacobi_eig3: a (N,3,3) symmetric -> (diagonalised a, eigenvectors as columns); 12 cyclic sweeps"""
    a = np.array(a, np.float64)
    N = a.shape[0]
    v = np.broadcast_to(np.eye(3), (N, 3, 3)).copy()
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        for _ in range(12):
            for p in range(2):
                for q in range(p + 1, 3):
                    apq = a[:, p, q]
                    skip = np.abs(apq) < 1e-300             # the kernel's `continue` (an identity rotation here)
                    th = (a[:, q, q] - a[:, p, p]) / (2.0 * apq)
                    tt = np.where(th >= 0, 1.0, -1.0) / (np.abs(th) + np.sqrt(th * th + 1.0))
                    c = 1.0 / np.sqrt(tt * tt + 1.0)
                    s = tt * c
                    c, s = np.where(skip, 1.0, c)[:, None], np.where(skip, 0.0, s)[:, None]
                    akp, akq = a[:, :, p].copy(), a[:, :, q].copy()
                    a[:, :, p], a[:, :, q] = c * akp - s * akq, s * akp + c * akq
                    apk, aqk = a[:, p, :].copy(), a[:, q, :].copy()
                    a[:, p, :], a[:, q, :] = c * apk - s * aqk, s * apk + c * aqk
                    vkp, vkq = v[:, :, p].copy(), v[:, :, q].copy()
                    v[:, :, p], v[:, :, q] = c * vkp - s * vkq, s * vkp + c * vkq
    return a, v


def _eig_sorted(H):
    """V (columns v_k) and lambda_k of H^T H, eigenvalues descending (numpy's singular-value order)"""
    B = np.einsum('nki,nkj->nij', H, H)
    d, V = jacobi_eig3(B)
    lam = np.diagonal(d, axis1=1, axis2=2)
    order = np.argsort(-lam, axis=1, kind='stable')
    return np.take_along_axis(V, order[:, None, :], axis=2), np.take_along_axis(lam, order, axis=1)


def _det3(m):
    return (m[:, 0, 0] * (m[:, 1, 1] * m[:, 2, 2] - m[:, 1, 2] * m[:, 2, 1])
            - m[:, 0, 1] * (m[:, 1, 0] * m[:, 2, 2] - m[:, 1, 2] * m[:, 2, 0])
            + m[:, 0, 2] * (m[:, 1, 0] * m[:, 2, 1] - m[:, 1, 1] * m[:, 2, 0]))


def _proper(U, s, V):
    """det(V) det(U) < 0: flip the last singular direction (loss.py:39-43); R = V U^T"""
    flip = _det3(V) * _det3(U) < 0
    V[flip, :, 2] *= -1
    s[flip, 2] *= -1
    return np.einsum('nik,njk->nij', V, U), s


def rotation_pre_fix(H):
    """the routine before the fix: U[:, k] = H v_k / sqrt(lambda_k), u2 by a cross product only when s2 <= 1e-9 s0"""
    H = np.asarray(H, np.float64)
    V, lam = _eig_sorted(H)
    s = np.sqrt(np.fmax(lam, 0.0))
    HV = np.einsum('nij,njk->nik', H, V)
    U = np.empty_like(H)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        for k in range(2):
            U[:, :, k] = HV[:, :, k] / np.fmax(s[:, k], 1e-300)[:, None]
        cr = np.cross(U[:, :, 0], U[:, :, 1])
        U[:, :, 2] = np.where((s[:, 2] > 1e-9 * s[:, 0])[:, None], HV[:, :, 2] / s[:, 2:3], cr)
    return _proper(U, s, V)


def _unit_orthogonal(u):
    """a unit vector orthogonal to u (unit): u x e_m, e_m the axis of u's smallest component"""
    m = np.argmin(np.abs(u), axis=1)
    e = np.eye(3)[m]
    w = np.cross(u, e)
    return w / np.sqrt((w * w).sum(1, keepdims=True))


def rotation(H):
    """the fixed routine: u0 = H v0 / |H v0|; u1 = H v1 Gram-Schmidt'ed against u0 (two passes) and normalised, any unit
    vector orthogonal to u0 when that is noise; u2 = sign((H v2).(u0 x u1)) u0 x u1, + at noise level;
    s_k = u_k^T H v_k.  Returns (R, s) with det(R) = +1."""
    H = np.asarray(H, np.float64)
    V, _ = _eig_sorted(H)
    HV = np.einsum('nij,njk->nik', H, V)
    w0 = HV[:, :, 0]
    n0 = np.sqrt((w0 * w0).sum(1))
    with np.errstate(divide='ignore', invalid='ignore'):
        u0 = np.where((n0 > 0)[:, None], w0 / n0[:, None], np.array([1.0, 0.0, 0.0]))
        w1 = HV[:, :, 1].copy()
        for _ in range(2):
            w1 = w1 - (u0 * w1).sum(1, keepdims=True) * u0
        n1 = np.sqrt((w1 * w1).sum(1))
        u1 = np.where((n1 > NOISE * n0)[:, None], w1 / n1[:, None], _unit_orthogonal(u0))
    c = np.cross(u0, u1)
    d = (HV[:, :, 2] * c).sum(1)
    sg = np.where((d < 0) & (-d > NOISE * n0), -1.0, 1.0)
    U = np.stack([u0, u1, sg[:, None] * c], axis=2)
    s = np.stack([n0, (u1 * HV[:, :, 1]).sum(1), sg * d], axis=1)
    return _proper(U, s, V)


def cross_covariance(pred, tgt):
    """the kernel's front half: centroids, norms and H = X0^T Y0 of the normalised, centred frames (loss.py:21-33)"""
    Y, X = np.asarray(pred, np.float64), np.asarray(tgt, np.float64)
    muX, muY = X.mean(1, keepdims=True), Y.mean(1, keepdims=True)
    X0, Y0 = X - muX, Y - muY
    nX = np.sqrt((X0 ** 2).sum((1, 2)))[:, None, None]
    nY = np.sqrt((Y0 ** 2).sum((1, 2)))[:, None, None]
    with np.errstate(divide='ignore', invalid='ignore'):
        H = np.einsum('nji,njk->nik', X0 / nX, Y0 / nY)
    return H, muX, muY, nX, nY


KINDS = ('ordinary', 'h36m', 'planar_pred', 'planar_tgt', 'planar_tgt_rot', 'collinear_tgt', 'collinear_pred',
         'collinear_both', 'reflected', 'rotated_copy', 'symmetric')


def _rot(rs):
    q, r = np.linalg.qr(rs.standard_normal((3, 3)))
    q = q * np.sign(np.diag(r))
    return q if np.linalg.det(q) > 0 else -q


def frames(kind, N, J, seed):
    """(pred, tgt) float32 (N,J,3) of one kind:
    ordinary        full rank, the target a rotated, scaled, noisy copy
    h36m            0.25 m spread about a centroid metres away, the prediction 3 cm off
    planar_pred     prediction in z = 0 (rank(H) = 2)
    planar_tgt      target in z = 0 (rank(H) = 2)
    planar_tgt_rot  target in a random plane, rounded to float32 (rank 2 up to that rounding)
    collinear_*     target, prediction or both on a random line (rank(H) = 1)
    reflected       the target is the mirrored prediction (the det(R) = -1 branch)
    rotated_copy    the target is a rotated, scaled, shifted copy (error 0 up to rounding)
    symmetric       octahedron (J >= 6) or triangle vertices, the rest at their centre: repeated singular values"""
    rs = np.random.RandomState(seed)
    f64 = np.float64
    if kind == 'ordinary':
        p = rs.standard_normal((N, J, 3))
        t = p @ _rot(rs) * 0.7 + 0.05 * rs.standard_normal((N, J, 3))
    elif kind == 'h36m':
        t = 0.25 * rs.standard_normal((N, J, 3)) + rs.uniform(-3, 3, (N, 1, 3)) + np.array([0, 0, 5.0])
        p = t + 0.03 * rs.standard_normal((N, J, 3))
    elif kind in ('planar_pred', 'planar_tgt'):
        p, t = rs.standard_normal((N, J, 3)), rs.standard_normal((N, J, 3))
        (p if kind == 'planar_pred' else t)[:, :, 2] = 0
    elif kind == 'planar_tgt_rot':
        t = rs.standard_normal((N, J, 3))
        t[:, :, 2] = 0
        t = t @ _rot(rs) + rs.standard_normal((N, 1, 3))
        p = t @ _rot(rs) + 0.3 * rs.standard_normal((N, J, 3))
    elif kind.startswith('collinear'):
        line = lambda: rs.standard_normal((N, J, 1)) * rs.standard_normal((N, 1, 3)) + rs.standard_normal((N, 1, 3))  # noqa
        p, t = rs.standard_normal((N, J, 3)), rs.standard_normal((N, J, 3))
        if kind in ('collinear_tgt', 'collinear_both'):
            t = line()
        if kind in ('collinear_pred', 'collinear_both'):
            p = line()
    elif kind == 'reflected':
        p = rs.standard_normal((N, J, 3))
        t = p * np.array([-1.0, 1.0, 1.0]) + 0.01 * rs.standard_normal((N, J, 3))
    elif kind == 'rotated_copy':
        p = rs.standard_normal((N, J, 3))
        t = 1.7 * p @ _rot(rs) + rs.standard_normal((N, 1, 3))
    elif kind == 'symmetric':
        base = np.concatenate([np.eye(3), -np.eye(3)]) if J >= 6 else np.array(
            [[1.0, 0, 0], [-0.5, 0.75 ** 0.5, 0], [-0.5, -0.75 ** 0.5, 0]])
        b = np.zeros((J, 3), f64)
        k = J // len(base)
        b[:k * len(base)] = np.tile(base, (k, 1))
        t = np.broadcast_to(b, (N, J, 3)) + rs.standard_normal((N, 1, 3))
        p = np.stack([b @ _rot(rs) for _ in range(N)]) * 0.8
    else:
        raise ValueError(kind)
    return np.asarray(p, np.float32), np.asarray(t, np.float32)


def spread(tgt):
    """(N,) the target's RMS distance from its centroid, the scale of the per-frame error bars"""
    X = np.asarray(tgt, np.float64)
    return np.sqrt(((X - X.mean(1, keepdims=True)) ** 2).sum(-1).mean(-1))


def p_mpjpe_per_frame(pred, tgt, routine=rotation):
    """(N,J,3) x2 -> (N,) the kernel's per-frame error with the given 3x3 routine"""
    Y, X = np.asarray(pred, np.float64), np.asarray(tgt, np.float64)
    H, muX, muY, nX, nY = cross_covariance(Y, X)
    R, s = routine(H)
    with np.errstate(divide='ignore', invalid='ignore'):
        a = s.sum(1)[:, None, None] * nX / nY
        aligned = a * (Y @ R) + (muX - a * (muY @ R))
    return np.sqrt(((aligned - X) ** 2).sum(-1)).mean(-1)
