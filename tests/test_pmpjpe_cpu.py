"""CPU: p_mpjpe_kernel's 3x3 alignment (numpy port, tests/pmpjperef.py) against np.linalg.svd (the fp64 oracle of
common/loss.py:14-53) on the frames where a Jacobi-on-H^T H SVD goes wrong: planar and collinear targets and
predictions, reflections, exact copies, repeated singular values, and scales from 1e-6 to 1e6.  The routine the
kernel used before is run on the same frames to show they reach its failure."""
import numpy as np
import pytest

import pmpjperef as PR
from conftest import load_golden
from oracle import pipeline_oracle as PO

JS = (3, 16, 17, 32)


def oracle_rotation(H):
    """R (with the det(R) = +1 fix of loss.py:39-43) from np.linalg.svd"""
    U, s, Vt = np.linalg.svd(H)
    V = np.swapaxes(Vt, 1, 2).copy()
    V[np.linalg.det(V @ np.swapaxes(U, 1, 2)) < 0, :, 2] *= -1
    return V @ np.swapaxes(U, 1, 2)


def check_rotation(R):
    RtR = np.einsum('nki,nkj->nij', R, R)
    assert np.abs(RtR - np.eye(3)).max() <= 1e-12
    assert np.abs(np.linalg.det(R) - 1).max() <= 1e-12


@pytest.mark.parametrize('J', JS)
@pytest.mark.parametrize('kind', PR.KINDS)
def test_port_matches_svd(kind, J):
    p, t = PR.frames(kind, 64, J, seed=J)
    R, s = PR.rotation(PR.cross_covariance(p, t)[0])
    check_rotation(R)
    got, ref = PR.p_mpjpe_per_frame(p, t), PO.p_mpjpe_per_frame(p, t)
    assert np.all(np.isfinite(got))
    assert np.all(np.abs(got - ref) <= 1e-8 * PR.spread(t)), np.abs(got - ref).max()
    if kind in ('rotated_copy', 'symmetric'):
        assert np.all(got <= 1e-6 * PR.spread(t))


@pytest.mark.parametrize('kind', ['planar_pred', 'planar_tgt', 'ordinary', 'reflected'])
def test_rank2_rotation_is_the_svd_one(kind):
    """with rank(H) >= 2 the proper rotation is unique: the port's R is the SVD's"""
    p, t = PR.frames(kind, 64, 17, seed=5)
    H = PR.cross_covariance(p, t)[0]
    R, s = PR.rotation(H)
    assert np.abs(R - oracle_rotation(H)).max() <= 1e-10
    sv = np.linalg.svd(H, compute_uv=False)
    assert np.abs(np.abs(s) - sv).max() <= 1e-12                  # s_k = u_k^T H v_k, up to the det sign of s_2


@pytest.mark.parametrize('scale', [1e-6, 1e-3, 1.0, 1e3, 1e6])
@pytest.mark.parametrize('kind', ['ordinary', 'planar_tgt', 'collinear_tgt', 'collinear_pred', 'reflected'])
def test_port_scale_invariant(kind, scale):
    p, t = PR.frames(kind, 32, 17, seed=11)
    p, t = (p * scale).astype(np.float32), (t * scale).astype(np.float32)
    R, _ = PR.rotation(PR.cross_covariance(p, t)[0])
    check_rotation(R)
    got, ref = PR.p_mpjpe_per_frame(p, t), PO.p_mpjpe_per_frame(p, t)
    assert np.all(np.abs(got - ref) <= 1e-8 * PR.spread(t))


def test_exact_copies():
    """rotated, scaled and shifted copies align to 0; a mirrored copy does not (R stays proper)"""
    rs = np.random.RandomState(3)
    p = rs.standard_normal((16, 17, 3))
    Q = np.linalg.qr(rs.standard_normal((3, 3)))[0]
    Q *= np.sign(np.linalg.det(Q))
    for t in (p, p @ Q, 3.5 * p @ Q + 2.0, 1e-4 * p @ Q):
        assert PR.p_mpjpe_per_frame(p, t).max() <= 1e-12 * max(1.0, PR.spread(t).max())
    t = p * np.array([1.0, -1.0, 1.0])
    got = PR.p_mpjpe_per_frame(p, t)
    assert np.all(got > 0.01) and np.all(np.abs(got - PO.p_mpjpe_per_frame(p, t)) <= 1e-12)


def test_port_matches_reference_golden():
    """the unmodified reference's own p_mpjpe (float32) on degenerate frames (tests/golden/make_golden_pmpjpe.py)"""
    G = load_golden('pmpjpe_degenerate')
    kinds = [k[:-len('_per_frame')] for k in G if k.endswith('_per_frame')]
    assert len(kinds) == 7
    for kind in kinds:
        p, t, ref = G[kind + '_pred'], G[kind + '_tgt'], G[kind + '_per_frame']
        assert np.abs(PR.p_mpjpe_per_frame(p, t) - ref).max() < 2e-5, kind      # the reference runs in float32
        assert np.abs(PO.p_mpjpe_per_frame(p, t) - ref).max() < 2e-5, kind


def test_zero_spread_is_nan():
    p, t = PR.frames('ordinary', 3, 17, seed=1)
    t[1] = t[1, 0]
    got = PR.p_mpjpe_per_frame(p, t)
    ref = PO.p_mpjpe_per_frame(p, t)
    assert np.isnan(got[1]) and np.isnan(ref[1])
    assert np.all(np.isfinite(got[[0, 2]])) and np.allclose(got[[0, 2]], ref[[0, 2]], rtol=1e-12)


@pytest.mark.parametrize('kind', ['planar_tgt', 'planar_tgt_rot', 'collinear_tgt', 'collinear_pred'])
def test_pre_fix_routine_fails_degenerate(kind):
    """the frames above do reach the old routine's failure: U = H V / sqrt(lambda) is not orthonormal there, so its R is
    no rotation and (but for a collinear prediction, whose distances do not see R's extra rows) the error is wrong"""
    p, t = PR.frames(kind, 200, 17, seed=0)
    H = PR.cross_covariance(p, t)[0]
    R, _ = PR.rotation_pre_fix(H)
    with np.errstate(invalid='ignore', over='ignore'):
        orth = np.abs(np.einsum('nki,nkj->nij', R, R) - np.eye(3)).max((1, 2))
        assert np.sum(~(orth <= 1e-6)) >= 20
        if kind != 'collinear_pred':
            old, ref = PR.p_mpjpe_per_frame(p, t, PR.rotation_pre_fix), PO.p_mpjpe_per_frame(p, t)
            assert np.sum(~(np.abs(old - ref) <= 1e-5 * ref)) >= 20
    assert np.all(np.abs(PR.p_mpjpe_per_frame(p, t) - PO.p_mpjpe_per_frame(p, t)) <= 1e-8 * PR.spread(t))
