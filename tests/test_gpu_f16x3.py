"""The fp32-grade inference form of the tensor-core core (three fp16 products on power-of-two-scaled operands,
csrc/gemm_tc.cuh) on the device, through gast_debug_gemm(core 0, tc_mode 0) and one whole model:
  * W = I: the output is (hi + lo) 2^-s_r of A exactly, bit for bit the emulated split (tests/f16x3ref.py);
  * every phase of the ring on rows spanning fp32's range, against fp64 at the fp32-grade bar, bitwise repeatable;
  * a model whose activations pass fp16's 65504 many times over matches the fp64 port at the parity bar."""
import numpy as np
import pytest
import torch

from gast_b200 import _lib, synth
from oracle import gast_oracle as O
import f16x3ref as F
import tf32ref as R

pytestmark = pytest.mark.gpu


def _gemm(A, W):
    lib = _lib.load()
    M, K = A.shape
    N = W.shape[0]
    a, w = torch.from_numpy(np.ascontiguousarray(A)).cuda(), torch.from_numpy(np.ascontiguousarray(W)).cuda()
    o = torch.full((M, N), float('nan'), dtype=torch.float32, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, 0, 0, None,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return o.cpu().numpy()


def test_device_split_is_f16x3ref_bit_for_bit():
    """W = identity (s_W = 14, W's hi exact and its lo zero): out = (hi + lo) 2^-s_r of A's row and stage"""
    M, K = 256, 64
    rs = np.random.RandomState(5)
    A = (rs.standard_normal((M, K)) * np.exp(rs.uniform(-20, 20, (M, K)))).astype(np.float32)
    A[:32] *= np.float32(1e-20)
    A[32:64] *= np.float32(1e20)
    assert np.isfinite(A).all()
    W = np.eye(K, dtype=np.float32)
    o = _gemm(A, W)
    h, lo, s = F.split_a(A, F.w_scale(W))
    emu = ((h.astype(np.float64) + lo.astype(np.float64)) * np.repeat(2.0 ** -s, F.KS, axis=1)).astype(np.float32)
    emu = emu + np.float32(0)                                  # the device's sum starts at +0
    assert np.array_equal(o.view(np.uint32), emu.view(np.uint32))


def _case(kind, rs, M, K):
    A = rs.standard_normal((M, K))
    if kind == 'range':
        A *= 10.0 ** rs.uniform(-30, 30, (M, 1))
    elif kind == 'mixed':
        A *= np.where(rs.uniform(size=(M, K)) < 0.5, 1e-6, 1e6)
    return A.astype(np.float32)


# every phase of a 3-, 4- or 5-slot ring: fewer stages than slots, one short, full, one wrap, two wraps, many
@pytest.mark.parametrize('stages', [1, 2, 3, 4, 5, 6, 7, 9, 11, 48])
@pytest.mark.parametrize('N', [4, 132, 256])
@pytest.mark.parametrize('kind', ['normal', 'range', 'mixed', 'wtiny', 'whuge'])
def test_f16x3_ring_phases(stages, N, kind):
    M, K = 300, 32 * stages                       # 300 rows: a partial last row tile
    rs = np.random.RandomState(1000 * stages + N)
    A = _case(kind, rs, M, K)
    wscale = {'wtiny': 1e-20, 'whuge': 1e20}.get(kind, 1.0)
    W = (rs.standard_normal((N, K)) / np.sqrt(K) * wscale).astype(np.float32)
    o1, o2 = _gemm(A, W), _gemm(A, W)
    ref = A.astype(np.float64) @ W.astype(np.float64).T
    assert np.isfinite(o1).all()
    # relative L2 per row (rows span up to 60 decades in 'range')
    rel = (np.linalg.norm(o1 - ref, axis=1) / np.linalg.norm(ref, axis=1)).max()
    assert rel < 2e-6, (stages, N, kind, rel)
    assert np.array_equal(o1, o2)


def test_non_finite_rows_become_nan():
    rs = np.random.RandomState(9)
    A = rs.standard_normal((128, 64)).astype(np.float32)
    A[1, 3] = np.inf
    A[2, 40] = np.nan
    o = _gemm(A, (rs.standard_normal((8, 64)) / 8).astype(np.float32))
    assert np.isnan(o[1]).all() and np.isnan(o[2]).all()
    assert np.isfinite(np.delete(o, [1, 2], axis=0)).all()


def test_activations_past_fp16_range():
    """one BatchNorm's gamma x 1e5: the block's activations reach ~1e5 - 1e6, past fp16's 65504; the form scales them
    instead of saturating and matches the fp64 port at the parity bar, relative to the output's size"""
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel
    J, fw, ch = 17, [3, 3, 3], 64
    m = SpatioTemporalModel(adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], [])), J, 2, J, fw,
                            channels=ch)
    synth.randomize_module(m, 3)
    with torch.no_grad():
        m.expand_bn.weight.mul_(1e5)
    p = {k: v.numpy() for k, v in m.state_dict().items()}
    x = synth.synth_input(3, 27, J, 2, seed=5)
    # the expand layer's output, the first GEMM's A: well past 65504
    si, ti = R.bn_fold(p, 'init_bn.')
    se, te = R.bn_fold(p, 'expand_bn.')
    w = p['expand_conv.weight'].astype(np.float64)[:, :, :, 0]
    xn = x.astype(np.float64) * si + ti
    h = sum(xn[:, k:k + 25] @ w[:, :, k].T for k in range(3)) * se + te
    assert np.maximum(h, 0).max() > 1e5
    ref = O.forward(x, p, O.adj_from_parents(synth.skeleton_parents(J)), fw)
    m = m.cuda().eval()
    with torch.no_grad():
        y = m(torch.from_numpy(x).cuda()).cpu().numpy()
    err = float(np.abs(y - ref).max() / np.abs(ref).max())
    assert np.isfinite(y).all() and err < 1e-5, err
