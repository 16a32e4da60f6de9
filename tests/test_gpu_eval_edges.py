"""GPU: the caller-side kernels of csrc/pipeline.cuh and the fused shrink + MPJPE epilogue against fp64, at the inputs
and sizes where they can go wrong.

- p_mpjpe_kernel: planar, collinear, reflected, symmetric and exact-copy frames (tests/pmpjperef.py::frames) at every
  joint count from 3 to 32 and 1 to 2^20 frames (4 frames per 128-thread block), one call mixing every kind, and the
  unmodified reference's own values on degenerate frames (tests/golden/pmpjpe_degenerate.npz).
- mpjpe_kernel: D = 1..4 around its 256-thread blocks and its 65,536-thread grid-stride loop, zero-distance rows,
  grad_scale != 1.
- shrink_mpjpe_kernel: more rows than its 1024 x 8 warps (several rows per warp), the 4096-clip batch, run-to-run and
  grid-to-grid repeatability.
- adam_multi_kernel (FusedAdam): with and without amsgrad and weight decay, tensors either side of a chunk boundary,
  and a state_dict resume.
"""
import ctypes as C
import io

import numpy as np
import pytest
import torch

import pmpjperef as PR
from conftest import load_golden
from gast_b200 import _lib as L
from gast_b200 import engine, synth
from gast_b200 import pipeline as P
from oracle import pipeline_oracle as PO

pytestmark = pytest.mark.gpu

PM_BAR = 2e-6          # per frame, times the target's RMS distance from its centroid


def _pm_dev(p, t):
    return P.p_mpjpe_per_frame(torch.from_numpy(p).cuda(), torch.from_numpy(t).cuda()).cpu().numpy().astype(np.float64)


def _pm_check(got, p, t, ref=None):
    ref = PO.p_mpjpe_per_frame(p, t) if ref is None else ref
    err = np.abs(got - ref)
    assert np.all(np.isfinite(got))
    assert np.all(err <= PM_BAR * PR.spread(t)), (err / PR.spread(t)).max()
    return (err / PR.spread(t)).max()


def _mixed(n_each, J, seed):
    """every kind of frame, n_each of each, shuffled; returns pred, tgt, kind index per frame"""
    ps, ts, ks = [], [], []
    for i, kind in enumerate(PR.KINDS):
        p, t = PR.frames(kind, n_each, J, seed=seed + i)
        ps.append(p), ts.append(t), ks.append(np.full(n_each, i))
    perm = np.random.RandomState(seed).permutation(n_each * len(PR.KINDS))
    return np.concatenate(ps)[perm], np.concatenate(ts)[perm], np.concatenate(ks)[perm]


@pytest.mark.parametrize('N', [1, 3, 4, 5, 1 << 20])
@pytest.mark.parametrize('J', [3, 15, 16, 17, 19, 31, 32])
def test_p_mpjpe_degenerate_frames(J, N, record_property):
    if N < 8:
        worst = 0.0
        for i, kind in enumerate(PR.KINDS):
            p, t = PR.frames(kind, N, J, seed=100 * J + 10 * N + i)
            worst = max(worst, _pm_check(_pm_dev(p, t), p, t))
        record_property('err_over_spread', worst)
        return
    # 2^20 frames: 4103 distinct ones (all kinds, shuffled) repeated; the oracle runs on the distinct frames
    p, t, _ = _mixed(373, J, seed=J)
    reps = -(-N // len(p))
    ref = np.tile(PO.p_mpjpe_per_frame(p, t), reps)[:N]
    pb, tb = np.tile(p, (reps, 1, 1))[:N], np.tile(t, (reps, 1, 1))[:N]
    got = _pm_dev(pb, tb)
    del pb
    record_property('err_over_spread', _pm_check(got, None, tb, ref))


def test_p_mpjpe_mixed_call_frames_independent(record_property):
    """one call over every kind plus two zero-spread frames: each frame equals its value from a call of its own kind
    bit for bit, the zero-spread frames are NaN (the reference divides by their zero norm) and leak into no neighbour"""
    J = 17
    p, t, k = _mixed(9, J, seed=7)
    p, t, k = np.concatenate([p[:5], p[:1], p[5:]]), np.concatenate([t[:5], t[:1], t[5:]]), np.insert(k, 5, k[0])
    t[5] = t[5, 3]                                          # target with zero spread, frame 5 of block 1
    p[-1] = p[-1, 0]                                        # prediction with zero spread, the last frame
    got = _pm_dev(p, t)
    assert np.isnan(got[5]) and np.isnan(got[-1])
    ref = PO.p_mpjpe_per_frame(p, t)
    assert np.isnan(ref[5]) and np.isnan(ref[-1])
    keep = np.ones(len(p), bool)
    keep[[5, -1]] = False
    record_property('err_over_spread', _pm_check(got[keep], p[keep], t[keep], ref[keep]))
    for i in range(len(PR.KINDS)):
        sel = keep & (k == i)
        alone = _pm_dev(np.ascontiguousarray(p[sel]), np.ascontiguousarray(t[sel]))
        assert np.array_equal(alone, got[sel]), PR.KINDS[i]


def test_p_mpjpe_reference_golden_degenerate(record_property):
    """the unmodified reference's p_mpjpe (float32) on degenerate frames, tests/golden/make_golden_pmpjpe.py"""
    G = load_golden('pmpjpe_degenerate')
    kinds = [k[:-len('_per_frame')] for k in G if k.endswith('_per_frame')]
    assert len(kinds) == 7
    worst = [0.0, 0.0]
    for kind in kinds:
        p, t = G[kind + '_pred'], G[kind + '_tgt']
        got = _pm_dev(p, t)
        err = np.abs(got - G[kind + '_per_frame']).max()
        assert err < 2e-5, kind                             # the reference itself runs in float32
        worst = [max(worst[0], err), max(worst[1], _pm_check(got, p, t))]
    record_property('err_vs_golden', worst[0])
    record_property('err_over_spread', worst[1])


def test_p_mpjpe_numpy_call_form_with_a_collinear_frame(record_property):
    """Protocol #2 over a set with one collapsed (collinear) detection stays finite and equals the fp64 mean"""
    from device.common.loss import p_mpjpe
    p, t = PR.frames('h36m', 64, 17, seed=3)
    pc, tc = PR.frames('collinear_pred', 1, 17, seed=4)
    p[17] = pc[0]
    pc, tc = PR.frames('collinear_tgt', 1, 17, seed=5)
    t[40] = tc[0]
    v = float(p_mpjpe(p, t))
    ref = PO.p_mpjpe_per_frame(p, t).mean()
    assert np.isfinite(v)
    record_property('err_mean', abs(v - ref))
    assert abs(v - ref) <= PM_BAR * PR.spread(t).max() + 1e-6 * ref, (v, ref)


# ------------------------------------------------------------------------------------------------
# mpjpe_kernel
# ------------------------------------------------------------------------------------------------
def _gast_mpjpe(pred, tgt, D, grad_scale, want_grad=True):
    p, t = torch.from_numpy(pred).cuda(), torch.from_numpy(tgt).cuda()
    loss = torch.empty((), dtype=torch.float32, device='cuda')
    dp = torch.empty_like(p) if want_grad else None
    rc = L.load().gast_mpjpe(C.c_void_p(p.data_ptr()), C.c_void_p(t.data_ptr()), p.numel() // D, D,
                             C.c_void_p(loss.data_ptr()), C.c_void_p(dp.data_ptr() if want_grad else 0), grad_scale,
                             C.c_void_p(P._mpjpe_ws(p.device).data_ptr()), C.c_void_p(engine._stream(p.device)))
    assert rc == 0, L.last_error()
    return loss.item(), (dp.cpu().numpy() if want_grad else None)


@pytest.mark.parametrize('n', [1, 255, 256, 257, 65535, 65536, 65537, 3 * 65536 + 5])
@pytest.mark.parametrize('D', [1, 2, 3, 4])
def test_mpjpe_sizes_and_dims(D, n, record_property):
    rs = np.random.RandomState(D * 1000 + n % 997)
    pred = rs.standard_normal((n, D)).astype(np.float32)
    tgt = rs.standard_normal((n, D)).astype(np.float32)
    zero = np.arange(3, n, 7)
    tgt[zero] = pred[zero]                                  # rows at zero distance: gradient 0, not NaN
    gs = 2.5
    loss, grad = _gast_mpjpe(pred, tgt, D, gs)
    rl, rg = PO.mpjpe(pred, tgt)
    record_property('loss_rel', abs(loss - rl) / rl)
    record_property('grad_err_times_n_over_gs', np.abs(grad - gs * rg).max() * n / gs)
    assert abs(loss - rl) <= 1e-6 * rl, (loss, rl)
    assert np.abs(grad - gs * rg).max() <= 1e-6 * gs / n, np.abs(grad - gs * rg).max() * n / gs
    assert np.all(grad[zero] == 0)
    loss_only, _ = _gast_mpjpe(pred, tgt, D, gs, want_grad=False)
    assert loss_only == loss


# ------------------------------------------------------------------------------------------------
# shrink_mpjpe_kernel (engine.run_model_mpjpe), the headline model: 27 frames, 17 joints, 128 channels
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def headline():
    from model.gast_net import SpatioTemporalModel
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    m = SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], channels=128)
    synth.randomize_module(m, 3)
    return m.cuda().eval()


def _fused(m, B, seed):
    x = torch.from_numpy(synth.synth_input(B, 27, 17, 2, seed=seed)).cuda()
    tgt = torch.from_numpy(synth.synth_target(B, 17, seed=seed + 1)).cuda()
    with torch.no_grad():
        y, loss = engine.run_model_mpjpe(m, x, tgt)
        y_plain = m(x)
    return x, tgt, y, loss.item(), y_plain


@pytest.mark.parametrize('B', [482, 483, 4096])
def test_fused_shrink_mpjpe_several_rows_per_warp(headline, B, record_property):
    """B * 17 > 1024 blocks x 8 warps = 8192 rows: each warp takes two or more rows"""
    x, tgt, y, loss, y_plain = _fused(headline, B, seed=B)
    assert B * 17 > 8192
    assert torch.equal(y, y_plain)
    ref = np.linalg.norm(y.cpu().numpy().astype(np.float64) - tgt.cpu().numpy(), axis=-1).mean()
    record_property('loss_rel', abs(loss - ref) / ref)
    assert abs(loss - ref) <= 1e-6 * ref, (loss, ref)
    with torch.no_grad():
        for _ in range(2):
            assert engine.run_model_mpjpe(headline, x, tgt)[1].item() == loss


def test_fused_shrink_mpjpe_alternating_grids(headline):
    """37 clips (79 blocks) and 483 clips (1024 blocks) in turn: each repeats its loss exactly, so the last block's
    ticket is back at 0 after every call"""
    runs = {B: _fused(headline, B, seed=B) for B in (37, 483)}
    with torch.no_grad():
        for _ in range(3):
            for B, (x, tgt, _, loss, _) in runs.items():
                assert engine.run_model_mpjpe(headline, x, tgt)[1].item() == loss, B


# ------------------------------------------------------------------------------------------------
# adam_multi_kernel (FusedAdam)
# ------------------------------------------------------------------------------------------------
ADAM_SHAPES = [(1,), (4095,), (64, 64), (4097,), (3 * 4096 + 1,)]


def _adam_data(seed):
    rs = np.random.RandomState(seed)
    ps = [(0.5 * rs.standard_normal(sh)).astype(np.float32) for sh in ADAM_SHAPES]
    grads = [[(rs.standard_normal(sh) * (10.0 if step == 1 else 0.1)).astype(np.float32) for sh in ADAM_SHAPES]
             for step in range(10)]
    return ps, grads


def _adam_run(params, opt, grads, steps):
    for step in steps:
        for p, g in zip(params, grads[step]):
            p.grad = torch.from_numpy(g).cuda()
        opt.step()
        for g in opt.param_groups:
            g['lr'] *= 0.95                                 # trainval.py:162-164


@pytest.mark.parametrize('wd', [0.0, 1e-2])
@pytest.mark.parametrize('amsgrad', [True, False])
def test_fused_adam_against_fp64(amsgrad, wd, record_property):
    assert int(L.load().gast_adam_chunk()) == 4096
    ps, grads = _adam_data(seed=17 + int(amsgrad) + int(wd * 100))
    params = [torch.nn.Parameter(torch.from_numpy(p.copy()).cuda()) for p in ps]
    opt = P.FusedAdam(params, lr=1e-3, weight_decay=wd, amsgrad=amsgrad)
    _adam_run(params, opt, grads, range(10))
    for i, p0 in enumerate(ps):
        p = p0.astype(np.float64).ravel()
        m, v, vm = np.zeros_like(p), np.zeros_like(p), np.zeros_like(p)
        lr = 1e-3
        for step in range(10):
            PO.adam_step(p, grads[step][i].astype(np.float64).ravel(), m, v, vm, step + 1, lr, weight_decay=wd,
                         amsgrad=amsgrad)
            lr *= 0.95
        err = np.abs(params[i].detach().cpu().numpy().ravel() - p).max()
        record_property('err_%d' % i, err)
        assert err < 2e-6, (ADAM_SHAPES[i], err)

    # save after step 5, load into a fresh optimiser over fresh parameters, continue: bit for bit the same run
    params_b = [torch.nn.Parameter(torch.from_numpy(p.copy()).cuda()) for p in ps]
    opt_b = P.FusedAdam(params_b, lr=1e-3, weight_decay=wd, amsgrad=amsgrad)
    _adam_run(params_b, opt_b, grads, range(5))
    buf = io.BytesIO()
    torch.save({'params': [p.detach() for p in params_b], 'opt': opt_b.state_dict()}, buf)
    _adam_run(params_b, opt_b, grads, range(5, 10))           # the saved copy is a snapshot: the live run goes on
    buf.seek(0)
    saved = torch.load(buf)
    params_c = [torch.nn.Parameter(p.clone()) for p in saved['params']]
    opt_c = P.FusedAdam(params_c, lr=123.0, weight_decay=wd, amsgrad=amsgrad)
    opt_c.load_state_dict(saved['opt'])
    _adam_run(params_c, opt_c, grads, range(5, 10))
    for a, b, c in zip(params, params_b, params_c):
        assert torch.equal(a, b) and torch.equal(a, c)
