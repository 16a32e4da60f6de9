"""GPU: scoring lifted test sets on the device (gast_pose_metrics, device/common/loss.py euclidean_losses / pck / auc,
gast_b200.evaluation.evaluate_sequences):
  * the device distances, pck and auc against the unmodified reference's (tests/golden/make_golden_metrics.py);
  * the segment rows against tests/metricsref.py in fp64, the P-MPJPE column against gast_p_mpjpe per frame;
  * determinism: repeated calls, a segment alone, among others and permuted, and the stream layout of the lifting;
  * evaluate_sequences against the staged, unchanged main.evaluate per group (needs oracle/_ref/, skipped without);
  * zero_root, the half-model refusal, and every bad argument refused on the host before any launch.
"""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest
import torch

import delayedref as D
import metricsref as MR
from conftest import load_golden, REPO, PKG
from gast_b200 import _lib, engine
from gast_b200 import pipeline as P
from gast_b200.evaluation import evaluate_sequences, AUC_THRESHOLDS
from gast_b200.realtime import lift_sequences

pytestmark = pytest.mark.gpu

CASES = ('random', 'on_threshold', 'degenerate')
REF = os.path.join(REPO, 'oracle', '_ref')
REF = REF if os.path.exists(os.path.join(REF, 'main.py')) else None
# main.evaluate runs p_mpjpe as a float32 numpy SVD and mpjpe as a float32 torch reduction: its e1 / e2 are good to
# about 1e-6 relative (the 2e-5 absolute P-MPJPE bar of test_gpu_pipeline on unit-scale frames); its poses are the
# whole-sequence forward, within WHOLE_BAR (5e-6) of the streamed ones.  1e-5 covers both.
REF_RTOL = 1e-5


@pytest.fixture(scope='module')
def G():
    return load_golden('metrics_17')


def _cuda(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize('case', CASES)
def test_euclidean_losses_against_reference(G, case):
    from device.common.loss import euclidean_losses
    p, t = G[case + '_pred'], G[case + '_tgt']
    d = euclidean_losses(_cuda(p), _cuda(t)).cpu().numpy()
    assert d.shape == G[case + '_dist'].shape and d.dtype == np.float32
    assert np.array_equal(d, MR.distances(p, t))                           # bit for bit: the pinned, IEEE-rounded order
    assert np.array_equal(d, np.sqrt(G[case + '_dist_sq']))                 # the reference's squares, bit for bit
    assert _ulps(d, G[case + '_dist']).max() <= 1                           # torch's CPU sqrt is not correctly rounded
    assert np.array_equal(euclidean_losses(p, t).cpu().numpy(), d)         # numpy call form


@pytest.mark.parametrize('case', CASES)
def test_pck_and_auc_against_reference(G, case):
    from device.common.loss import pck, auc
    p, t = _cuda(G[case + '_pred']), _cuda(G[case + '_tgt'])
    for th, want in zip(G['thresholds'], G[case + '_pck']):
        got = pck(p, t, threshold=float(th))
        assert isinstance(got, float) and got == want, (th, got, want)      # exactly, on-threshold distances included
    assert pck(p, t) == G[case + '_pck'][list(G['thresholds']).index(150.0)]
    a = auc(p, t)
    assert isinstance(a, float)
    assert abs(a - float(G[case + '_auc'])) <= 1e-15 * abs(float(G[case + '_auc']))
    assert auc(G[case + '_pred'], G[case + '_tgt']) == a                   # numpy call form


def _frames(N, J, seed):
    rs = np.random.RandomState(seed)
    t = 0.25 * rs.standard_normal((N, J, 3)) + rs.uniform(-1, 1, (N, 1, 3))
    p = t + rs.uniform(0.005, 0.2, (N, 1, 1)) * rs.standard_normal((N, J, 3))
    return p.astype(np.float32), t.astype(np.float32)


THR = [0.0, 0.01, 0.05, 0.1, 0.15, 0.3]


@pytest.mark.parametrize('J', [3, 17, 19, 32])
@pytest.mark.parametrize('zero_root', [False, True])
def test_rows_against_metricsref(J, zero_root):
    lengths = [0, 1, 63, 64, 65, 200, 0, 517]
    seg = np.concatenate([[0], np.cumsum(lengths)])
    p, t = _frames(int(seg[-1]), J, seed=J)
    rows = P.pose_metrics(_cuda(p), _cuda(t), seg, THR, zero_root=zero_root).cpu().numpy()
    ref = MR.segment_rows(p, t, seg, THR, zero_root=zero_root)
    assert rows.shape == ref.shape == (len(lengths), 3 + J + len(THR))
    assert np.array_equal(rows[:, 0], ref[:, 0])
    assert np.array_equal(rows[:, 3 + J:], ref[:, 3 + J:])                  # counts exactly
    for c in [1] + list(range(3, 3 + J)):
        assert np.allclose(rows[:, c], ref[:, c], rtol=1e-12, atol=0), c
    assert np.allclose(rows[:, 2], ref[:, 2], rtol=1e-6, atol=0)             # port vs kernel, each rounded to float32
    tz = MR.zeroed(t) if zero_root else t
    pm = P.p_mpjpe_per_frame(_cuda(p), _cuda(tz)).cpu().numpy().astype(np.float64) if len(p) else np.zeros(0)
    want = np.array([pm[seg[s]:seg[s + 1]].sum() for s in range(len(lengths))])
    assert np.allclose(rows[:, 2], want, rtol=1e-12, atol=0)                 # gast_p_mpjpe per frame, summed in fp64
    assert np.all(rows[[0, 6]] == 0)


def test_zero_root_against_a_zeroed_copy():
    p, t = _frames(300, 17, seed=3)
    tt = _cuda(t)
    before = tt.clone()
    a = P.pose_metrics(_cuda(p), tt, [0, 120, 300], THR, zero_root=True)
    b = P.pose_metrics(_cuda(p), _cuda(MR.zeroed(t)), [0, 120, 300], THR, zero_root=False)
    assert torch.equal(a, b)
    assert torch.equal(tt, before)                                         # the caller's target is not written


def test_rows_are_deterministic_and_independent_of_the_other_segments():
    lengths = [700, 5, 130, 64, 2000, 1]
    seg = np.concatenate([[0], np.cumsum(lengths)])
    p, t = _frames(int(seg[-1]), 17, seed=9)
    pc, tc = _cuda(p), _cuda(t)
    thr = THR + AUC_THRESHOLDS
    rows = P.pose_metrics(pc, tc, seg, thr).cpu().numpy()
    assert np.array_equal(rows, P.pose_metrics(pc, tc, seg, thr).cpu().numpy(), equal_nan=True)
    for s in range(len(lengths)):                                          # alone
        a, b = seg[s], seg[s + 1]
        alone = P.pose_metrics(pc[a:b].contiguous(), tc[a:b].contiguous(), [0, b - a], thr).cpu().numpy()
        assert np.array_equal(alone[0].view(np.uint64), rows[s].view(np.uint64)), s
    perm = [4, 2, 0, 5, 3, 1]                                              # permuted
    pp = torch.cat([pc[seg[s]:seg[s + 1]] for s in perm])
    tp = torch.cat([tc[seg[s]:seg[s + 1]] for s in perm])
    sp = np.concatenate([[0], np.cumsum([lengths[s] for s in perm])])
    rp = P.pose_metrics(pp, tp, sp, thr).cpu().numpy()
    assert np.array_equal(rp.view(np.uint64), rows[perm].view(np.uint64))


def _lib_call(pred, tgt, N, J, seg, thr, rows, ws, wsb, procrustes=1):
    lib = _lib.load()
    seg = np.ascontiguousarray(seg, dtype=np.int64)
    thr = np.ascontiguousarray(thr, dtype=np.float32)
    return lib.gast_pose_metrics(C.c_void_p(pred), C.c_void_p(tgt), N, J, seg.ctypes.data_as(C.POINTER(C.c_int64)),
                                 len(seg) - 1, thr.ctypes.data_as(C.POINTER(C.c_float)), thr.size, 0, procrustes,
                                 C.c_void_p(rows), None, C.c_void_p(ws), wsb,
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream))


def test_bad_arguments_refused_before_any_launch():
    """each bad argument is refused on the host: the output rows keep their sentinel, and nothing was enqueued that
    could fault (the stream synchronises cleanly afterwards)"""
    lib = _lib.load()
    p, t = _frames(100, 17, seed=1)
    pc, tc = _cuda(p), _cuda(t)
    wsb = int(lib.gast_pose_metrics_workspace_bytes(2, 17, 2, 100))
    ws = torch.empty(wsb, dtype=torch.uint8, device='cuda')
    rows = torch.full((2, 3 + 17 + 2), -7.0, dtype=torch.float64, device='cuda')
    good = dict(pred=pc.data_ptr(), tgt=tc.data_ptr(), N=100, J=17, seg=[0, 40, 100], thr=[0.1, 0.2],
                rows=rows.data_ptr(), ws=ws.data_ptr(), wsb=wsb)
    bad = [dict(seg=[0, 60, 40]), dict(seg=[0, 40, 99]), dict(seg=[1, 40, 100]), dict(seg=[-5, 40, 100]),
           dict(thr=[0.1, float('nan')]), dict(J=33), dict(J=0), dict(N=-1, seg=[0, 40, -1]), dict(wsb=wsb - 1),
           dict(ws=None), dict(rows=None), dict(pred=None), dict(J=2, seg=[0, 40, 100])]
    for b in bad:
        kw = dict(good, **b)
        assert _lib_call(**kw) != 0, b
    assert _lib_call(**dict(good, thr=list(range(65)))) != 0               # more than 64 thresholds
    assert _lib.load().gast_pose_metrics_workspace_bytes(0, 17, 2, 100) == 0
    assert _lib.load().gast_pose_metrics_workspace_bytes(1, 17, 65, 100) == 0
    torch.cuda.synchronize()
    assert torch.all(rows == -7.0)                                          # refused before any launch
    assert _lib_call(**good) == 0
    torch.cuda.synchronize()
    assert not torch.any(rows == -7.0)
    with pytest.raises(engine.GastError, match='sorted'):
        P.pose_metrics(pc, tc, [0, 60, 40, 100], THR)
    with pytest.raises(engine.GastError, match='NaN'):
        P.pose_metrics(pc, tc, [0, 100], [float('nan')])
    with pytest.raises(engine.GastError, match='N,J,3'):
        P.pose_metrics(pc, tc[:50], [0, 50], THR)
    with pytest.raises(engine.GastError, match='Procrustes'):
        P.pose_metrics(pc[:, :2].contiguous(), tc[:, :2].contiguous(), [0, 100], THR)


# ------------------------------------------------------------------------------------------------
# evaluate_sequences
# ------------------------------------------------------------------------------------------------
def _test_set(J, causal, seed, lengths=(90, 31, 200, 7, 64, 150)):
    case = D.Case(J, (3, 3, 3), 32, 1, sum(lengths), 0, (), seed, causal, True)
    m = D.module(case, dilated=True).cuda()
    x = D.frames(case)[:, 0]
    cuts = np.cumsum([0] + list(lengths))
    rs = np.random.RandomState(seed)
    p2 = [x[cuts[k]:cuts[k + 1]] for k in range(len(lengths))]
    p3 = [(0.25 * rs.standard_normal((T, J, 3)) + rs.uniform(-1, 1, (1, 1, 3))).astype(np.float32) for T in lengths]
    groups = ['Walk', 'Sit', 'Walk', 'Eat', 'Sit', 'Walk'][:len(lengths)]
    return m, p2, p3, groups


@pytest.fixture(scope='module')
def main_module():
    """the staged, unchanged main.py (main.evaluate) with the drop-in package ahead of the reference root"""
    if REF is None:
        pytest.skip('reference caller files not staged (python oracle/make_ref.py <original checkout>)')
    saved_path, saved_mods = list(sys.path), dict(sys.modules)
    sys.path[:] = [PKG, REF] + [p for p in sys.path if p not in (PKG, REF)]
    sys.modules.pop('main', None)
    mn = importlib.import_module('main')
    gen = importlib.import_module('common.generators')
    yield mn, gen
    sys.path[:] = saved_path
    for name in list(sys.modules):
        if name not in saved_mods and name.split('.')[0] in ('main', 'tools'):
            sys.modules.pop(name, None)


@pytest.mark.parametrize('J,causal', [(17, False), (17, True), (19, False)])
@pytest.mark.parametrize('augment', [False, True])
def test_evaluate_sequences_against_main_evaluate(main_module, J, causal, augment, capsys):
    mn, gen = main_module
    m, p2, p3, groups = _test_set(J, causal, seed=20 + J + causal)
    kl, kr, jl, jr = D.symmetry(J)
    res = evaluate_sequences(m, p2, p3, groups, augment=augment, kps_left=kl, kps_right=kr, joints_left=jl,
                             joints_right=jr, n_streams=4, chunk=48)
    assert res.groups == ['Walk', 'Sit', 'Eat']
    pad = (m.receptive_field() - 1) // 2
    e1s, e2s = [], []
    for g in res.groups:
        idx = [i for i, x in enumerate(groups) if x == g]
        it = gen.UnchunkedGenerator(None, [p3[i] for i in idx], [p2[i] for i in idx], pad=pad,
                                    causal_shift=pad if causal else 0, augment=augment, kps_left=kl, kps_right=kr,
                                    joints_left=jl, joints_right=jr)
        e1, e2 = mn.evaluate(it, m, jl, jr, g)
        e1s.append(e1)
        e2s.append(e2)
        assert res[g].frames == sum(len(p3[i]) for i in idx)
        assert abs(res[g].mpjpe * 1000 - e1) <= REF_RTOL * e1, (g, res[g].mpjpe * 1000, e1)
        assert abs(res[g].p_mpjpe * 1000 - e2) <= REF_RTOL * e2, (g, res[g].p_mpjpe * 1000, e2)
    capsys.readouterr()
    a1, a2 = res.action_wise()
    assert abs(a1 * 1000 - np.mean(e1s)) <= REF_RTOL * np.mean(e1s)
    assert abs(a2 * 1000 - np.mean(e2s)) <= REF_RTOL * np.mean(e2s)


def test_evaluate_sequences_is_the_rows_of_its_lifted_poses():
    """the group sums are the rows of lift_sequences' poses against zeroed targets; pck / auc / per_joint follow"""
    m, p2, p3, groups = _test_set(17, False, seed=5)
    kl, kr, jl, jr = D.symmetry(17)
    res = evaluate_sequences(m, p2, p3, groups, augment=True, kps_left=kl, kps_right=kr, joints_left=jl,
                             joints_right=jr, thresholds=[0.2, 0.5])
    lifted = lift_sequences(m, p2, augment=True, kps_left=kl, kps_right=kr, joints_left=jl, joints_right=jr)
    for g in res.groups:
        idx = [i for i, x in enumerate(groups) if x == g]
        pred = np.concatenate([lifted[i].cpu().numpy() for i in idx])
        tgt = MR.zeroed(np.concatenate([p3[i] for i in idx]))
        d = MR.distances(pred, tgt).astype(np.float64)
        n = d.size
        assert np.isclose(res[g].mpjpe, d.mean(1).sum() / len(d), rtol=1e-12, atol=0)
        assert np.allclose(res[g].per_joint, d.sum(0) / len(d), rtol=1e-12, atol=0)
        d32 = MR.distances(pred, tgt)
        assert res[g].pck == (d32 < 150.0).sum() / n
        assert res[g].pck_at == {0.2: (d32 < np.float32(0.2)).sum() / n, 0.5: (d32 < np.float32(0.5)).sum() / n}
        want_auc = torch.tensor([(d32 < np.float32(th)).sum() / n for th in AUC_THRESHOLDS], dtype=torch.float64)
        assert res[g].auc == want_auc.mean().item()


def test_evaluate_sequences_deterministic_across_stream_layouts():
    m, p2, p3, groups = _test_set(17, True, seed=8)
    kl, kr, jl, jr = D.symmetry(17)
    kw = dict(augment=True, kps_left=kl, kps_right=kr, joints_left=jl, joints_right=jr, thresholds=True)
    base = evaluate_sequences(m, p2, p3, groups, **kw)
    for ns, ch in [(64, 256), (1, 16), (3, 100)]:
        r = evaluate_sequences(m, p2, p3, groups, n_streams=ns, chunk=ch, **kw)
        for g in base.groups:
            a, b = base[g], r[g]
            assert (a.frames, a.mpjpe, a.p_mpjpe, a.pck, a.auc) == (b.frames, b.mpjpe, b.p_mpjpe, b.pck, b.auc)
            assert np.array_equal(a.per_joint, b.per_joint)
    # a group alone scores the same bits as among the others
    idx = [i for i, g in enumerate(groups) if g == 'Sit']
    alone = evaluate_sequences(m, [p2[i] for i in idx], [p3[i] for i in idx], ['Sit'] * len(idx), **kw)['Sit']
    assert (alone.mpjpe, alone.p_mpjpe, alone.auc) == (base['Sit'].mpjpe, base['Sit'].p_mpjpe, base['Sit'].auc)


def test_evaluate_sequences_edges():
    m, p2, p3, _ = _test_set(17, False, seed=4, lengths=(40, 0, 25))
    before = [x.copy() for x in p3]
    res = evaluate_sequences(m, p2, p3, ['a', 'empty', 'a'])
    assert res['empty'].frames == 0 and np.isnan(res['empty'].mpjpe) and np.isnan(res['empty'].p_mpjpe)
    assert all(np.array_equal(a, b) for a, b in zip(p3, before))           # zero_root does not write the targets
    one = evaluate_sequences(m, p2, p3)
    assert one.groups == [None] and one[None].frames == 65
    with pytest.raises(engine.GastError, match='poses_3d'):
        evaluate_sequences(m, p2, [x[:, :16] for x in p3])


def test_half_model_refused_before_any_launch():
    m, p2, p3, _ = _test_set(17, False, seed=4, lengths=(40, 25))
    mh = m.half()
    with pytest.raises(engine.GastError, match='inference only'):
        evaluate_sequences(mh, p2, p3)


@pytest.mark.parametrize('precision', ['tf32', 'fp16'])
def test_evaluate_sequences_at_precision(precision):
    """the opt-in precisions score what lift_sequences lifts at them"""
    m, p2, p3, groups = _test_set(17, False, seed=6)
    engine.set_precision(m, precision)
    res = evaluate_sequences(m, p2, p3, groups)
    lifted = lift_sequences(m, p2)
    for g in res.groups:
        idx = [i for i, x in enumerate(groups) if x == g]
        pred = np.concatenate([lifted[i].cpu().numpy() for i in idx])
        d = MR.distances(pred, MR.zeroed(np.concatenate([p3[i] for i in idx]))).astype(np.float64)
        assert np.isclose(res[g].mpjpe, d.mean(1).sum() / len(d), rtol=1e-12, atol=0)
