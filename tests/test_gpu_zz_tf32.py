"""GPU: the opt-in single-pass TF32 precision (`gast_set_precision(h, 1)`, `engine.set_precision(model, 'tf32')`).

  * gast_debug_gemm with tc_mode 1: every phase of the 1xTF32 ring, weights scaled by 300, against the emulated
    tf32(A) . tf32(W) (fp32-accumulation level) and against exact fp64 (TF32 level); two runs bitwise equal; the
    device's operand rounding equals tests/tf32ref.tf32 bit for bit.
  * the sub-module kinds in TF32 against tests/tf32ref.py (tight) and exact fp64: the ratio shows the single TF32
    product.
  * the model forward in TF32 across joint counts, depths, widths, schedules and a ragged batch against tf32ref and
    against exact fp64 (the documented bar); see the bars below for why the model-level match is looser.
  * switching leaves nothing behind; the streams follow the model's setting; the refusals; launch counts.
Measured errors go to $GAST_TEST_REPORT_DIR/tf32.txt when that is set.
"""
import copy
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from gast_b200 import _lib, engine, synth, tta
from gast_b200.realtime import CausalStream, PoseStream, lift_sequences
from oracle import gast_oracle as O
import tf32ref as R

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')

# The device and tests/tf32ref.py round the same operands, but from activations that differ in the last fp32 bits; a
# rare operand then lands on the other side of a TF32 rounding boundary and moves its outputs by up to ~1e-4 (this
# sets the max-norm distance, so the emulation is compared in relative L2).  Through one layer that stays rare: the
# sub-modules match the emulation to 1e-7 - 7e-6 in L2 against 2e-4 - 4e-4 from fp64.  Through a whole model the
# moved outputs are the next layer's operands and move their roundings in turn, so the device's distance from the
# emulation grows to a fraction of the rounding effect itself: measured 2.8e-4 - 5.3e-4 in L2 (1.9e-3 for the
# 5-stage model) against 4.3e-4 - 2.2e-3 from fp64, ratios 1.1 - 2.6.  A 3xTF32 result sits 1e-6 from fp64, i.e. at
# ratio ~0.  H100 80GB HBM3, one run; the bars are ~4x those measurements.
MOD_L2_BAR = 3e-5     # ||y - y_tf32ref|| / ||y||, sub-modules
MOD_RATIO = 20.0      # sub-modules: L2 vs fp64 / L2 vs tf32ref (measured 47 - 3000)
MODEL_L2_BAR = 2.5e-3  # ||y - y_tf32ref|| / ||y||, whole models
MODEL_RATIO = 1.0     # whole models: closer to the single-product emulation than to fp64
TF32_FLOOR = 1e-4     # L2 vs fp64 of a TF32 forward: the single product's rounding is there (3xTF32: ~1e-6)
EXACT_BAR = 5e-3      # max |y - y64| / max |y|: TF32 against exact fp64 (DESIGN.md §4.1, the documented bar)
STREAM_L2_BAR = 1e-3  # ||y - y_whole|| / ||y_whole|| in TF32: stream against the whole-sequence forward (2.6e-4)


def report(line):
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        with open(os.path.join(REPORT_DIR, 'tf32.txt'), 'a') as f:
            f.write(line + '\n')


def _adj(J):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))


def _masks(J):
    return O.local_masks(O.adj_from_parents(synth.skeleton_parents(J)))


def _handle(m):
    return list(m.__dict__['_gast_handles'].values())[0]


def _tc_launches(m):
    h = _handle(m)
    return int(h.lib.gast_last_tc_launch_count(h.h))


def _model(J, fw, ch, strided=False, causal=False, dense=False, seed=11):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    if strided:
        m = SpatioTemporalModelOptimized1f(_adj(J), J, 2, J, list(fw), causal=causal, dropout=0.05, channels=ch)
    else:
        m = SpatioTemporalModel(_adj(J), J, 2, J, list(fw), causal=causal, dropout=0.05, channels=ch, dense=dense)
    synth.randomize_module(m, seed)
    return m.eval()


def _rel(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())


def _l2(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))


# ------------------------------------------------------------------------------------------------------------------
# one GEMM (gast_debug_gemm, tc_mode 1)
# ------------------------------------------------------------------------------------------------------------------
def _gemm(a, w, M, N, K, tc_mode=1):
    lib = _lib.load()
    o = torch.full((M, N), float('nan'), dtype=torch.float32, device='cuda')
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, tc_mode, 0, None,
                             torch.cuda.current_stream().cuda_stream)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return o.cpu().numpy()


# every phase of a 3-, 4- or 5-slot ring: fewer stages than slots, one short, full, one wrap, two wraps, many
@pytest.mark.parametrize('stages', [1, 2, 3, 4, 5, 6, 7, 9, 11, 48])
@pytest.mark.parametrize('N', [4, 132, 256])
@pytest.mark.parametrize('wscale', [None, 300.0])
def test_tf32_gemm_ring_phases(stages, N, wscale):
    M, K = 300, 32 * stages                       # 300 rows: a partial last row tile
    rs = np.random.RandomState(1000 * stages + N)
    A = rs.standard_normal((M, K)).astype(np.float32)
    W = (rs.standard_normal((N, K)) * (wscale or 1.0 / np.sqrt(K))).astype(np.float32)
    a, w = torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda()
    o1 = _gemm(a, w, M, N, K)
    o2 = _gemm(a, w, M, N, K)
    emu = R.tf32(A).astype(np.float64) @ R.tf32(W).astype(np.float64).T
    exact = A.astype(np.float64) @ W.astype(np.float64).T
    l2 = lambda d, r: float(np.sqrt((d ** 2).mean() / (r ** 2).mean()))   # noqa: E731
    e_emu, e_exact = l2(o1 - emu, emu), l2(o1 - exact, exact)
    report('gemm stages %d N %d wscale %s: rel L2 vs emulated %.2e, vs exact %.2e' % (stages, N, wscale, e_emu, e_exact))
    assert np.isfinite(o1).all()
    assert e_emu < 2e-6, e_emu                    # fp32 accumulation of the exact tf32 products
    assert 5e-5 < e_exact < 1e-3, e_exact         # TF32 operand rounding
    assert np.array_equal(o1, o2)


def test_device_operand_rounding_is_tf32ref_bit_for_bit():
    """W = identity: out = tf32(A) . 1 exactly, so the output shows the device's cvt.rna.tf32.f32 of A"""
    M, K = 256, 32
    rs = np.random.RandomState(5)
    A = (rs.standard_normal((M, K)) * np.exp(rs.uniform(-20, 20, (M, K)))).astype(np.float32)
    u = A.view(np.uint32)
    u[:64] = (u[:64] & np.uint32(0xFFFFE000)) | np.uint32(0x1000)      # exact ties, both signs
    u[64:96] = (u[64:96] & np.uint32(0xFFFFE000)) | np.uint32(0x0FFF)  # just below a tie
    W = np.eye(K, dtype=np.float32)
    o = _gemm(torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda(), M, K, K)
    assert np.array_equal(o.view(np.uint32), R.tf32(A).view(np.uint32))


def test_debug_gemm_refuses_bad_modes():
    lib = _lib.load()
    a = torch.zeros((128, 32), device='cuda')
    w = torch.zeros((32, 32), device='cuda')
    o = torch.zeros((128, 32), device='cuda')
    st = torch.cuda.current_stream().cuda_stream
    for core, mode in ((0, 2), (0, -1), (1, 1)):
        assert lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), 128, 32, 32, core, mode, 0, None, st) != 0
        assert 'tc_mode' in _lib.last_error()


# ------------------------------------------------------------------------------------------------------------------
# the model
# ------------------------------------------------------------------------------------------------------------------
MODELS = [  # J, fw, ch, strided, causal, dense, B, T
    (17, (3, 3, 3), 128, True, False, False, 5, 27),
    (17, (3, 3, 3), 128, False, False, False, 3, 40),
    (15, (3, 3, 3), 32, False, False, False, 3, 29),
    (16, (3, 3, 3), 64, False, True, False, 2, 33),
    (19, (3, 3), 256, True, False, False, 7, 9),
    (17, (5, 3, 3), 64, True, True, False, 3, 45),
    (17, (3, 3, 3, 3, 3), 32, True, False, False, 2, 243),
    (17, (3, 3, 3, 3), 64, False, True, False, 13, 90),
    (17, (3, 3, 3), 32, False, False, True, 4, 28),
    (19, (3, 5), 96, False, False, False, 11, 17),
]


def _tf32_case(J, fw, ch, strided, causal, dense, B, T):
    m = _model(J, fw, ch, strided, causal, dense)
    p = {k: v.numpy() for k, v in m.state_dict().items()}
    x = synth.synth_input(B, T, J, 2, seed=7 + B)
    sched_strided = strided or (T == m.receptive_field() and not dense)
    emu, gem = R.forward(x, p, _masks(J), fw, causal, sched_strided, dense, rnd=True)
    exact, _ = R.forward(x, p, _masks(J), fw, causal, sched_strided, dense, rnd=False)
    m = engine.set_precision(m.cuda(), 'tf32')
    with torch.no_grad():
        y = m(torch.from_numpy(x).cuda()).cpu().numpy()
    return m, y, emu, exact, gem


@pytest.mark.parametrize('J,fw,ch,strided,causal,dense,B,T', MODELS)
def test_model_forward_computes_the_single_tf32_product(J, fw, ch, strided, causal, dense, B, T):
    m, y, emu, exact, gem = _tf32_case(J, fw, ch, strided, causal, dense, B, T)
    assert y.shape == emu.shape
    assert gem.tc == gem.count and _tc_launches(m) == gem.tc        # every GEMM on the tensor cores
    l_emu, l_exact, e_exact = _l2(y, emu), _l2(y, exact), _rel(y, exact)
    report('model J%d fw%s c%d strided %d causal %d dense %d B%d T%d: L2 vs tf32ref %.2e, vs fp64 %.2e (ratio %.1f); '
           'max vs tf32ref %.2e, vs fp64 %.2e' % (J, fw, ch, strided, causal, dense, B, T, l_emu, l_exact,
                                                  l_exact / max(l_emu, 1e-12), _rel(y, emu), e_exact))
    assert l_emu < MODEL_L2_BAR, l_emu
    assert e_exact < EXACT_BAR, e_exact
    assert l_exact > TF32_FLOOR, l_exact
    assert l_exact > MODEL_RATIO * l_emu, (l_exact, l_emu)


MODULES = [('mod_block_17_32', 'block'), ('mod_block_19_16', 'block'), ('mod_local_17_32', 'local'),
           ('mod_mglobal_17_32', 'mglobal'), ('mod_global_17_32', 'global'), ('mod_semch_17_32', 'semch'),
           ('mod_semgc_17_32', 'semgc')]


def _module(kind, J, C):
    from model.gast_net import GraphAttentionBlock
    from model.local_attention import LocalGraph, SemCHGraphConv, local_adjacencies
    from model.global_attention import MultiGlobalGraph, GlobalGraph
    from model.sem_graph_conv import SemGraphConv
    if kind == 'block':
        return GraphAttentionBlock(_adj(J), C, C, 0.05)
    if kind == 'local':
        return LocalGraph(_adj(J), C, C, 0.05)
    if kind == 'mglobal':
        return MultiGlobalGraph(_adj(J), C, C // 4, dropout=0.05)
    if kind == 'global':
        return GlobalGraph(_adj(J), C, C // 4)
    _, con = local_adjacencies(_adj(J))
    return SemCHGraphConv(C, C, con) if kind == 'semch' else SemGraphConv(C, C, con, bias=True)


@pytest.mark.parametrize('name,kind', MODULES)
def test_module_kinds_in_tf32(name, kind):
    g = load_golden(name)
    meta = g['meta']
    mod = _module(kind, meta['J'], meta['C'])
    synth.randomize_module(mod, meta['seed'])
    mod = mod.cuda().eval()
    p = {k: v.cpu().numpy() for k, v in mod.state_dict().items()}
    masks = g['mask'].astype(bool) if kind in ('semch', 'semgc') else _masks(meta['J'])
    xin = g['x'].transpose(0, 3, 1, 2) if kind == 'block' else g['x']
    emu, gem = R.module_forward(kind, xin, p, masks, rnd=True)
    exact, _ = R.module_forward(kind, xin, p, masks, rnd=False)
    engine.set_precision(mod, 'tf32')
    with torch.no_grad():
        y = mod(torch.from_numpy(np.ascontiguousarray(xin)).cuda()).cpu().numpy()
    l_emu, l_exact, e_exact = _l2(y, emu), _l2(y, exact), _rel(y, exact)
    report('module %s: L2 vs tf32ref %.2e, vs fp64 %.2e; max vs tf32ref %.2e, vs fp64 %.2e; tc %d of %d'
           % (name, l_emu, l_exact, _rel(y, emu), e_exact, gem.tc, gem.count))
    assert _tc_launches(mod) == gem.tc
    assert l_emu < MOD_L2_BAR, l_emu
    assert e_exact < EXACT_BAR, e_exact
    if gem.tc:
        assert l_exact > MOD_RATIO * l_emu, (l_exact, l_emu)


# ------------------------------------------------------------------------------------------------------------------
# switching, schedules, launch counts
# ------------------------------------------------------------------------------------------------------------------
def test_switching_leaves_nothing_behind():
    m = _model(17, (3, 3, 3), 64).cuda()
    xs = [torch.from_numpy(synth.synth_input(6, T, 17, 2, seed=T)).cuda() for T in (27, 40)]

    def run():
        with torch.no_grad():
            out = [m(x).cpu().numpy() for x in xs]
        return out, m._gast_last_launches, _tc_launches(m)

    a, la, ta = run()
    assert engine.get_precision(m) == 'fp32'
    engine.set_precision(m, 'tf32')
    assert all(engine.get_precision(s) == 'tf32' for s in m.modules())
    t, lt, tt = run()
    engine.set_precision(m, 'fp32')
    b, lb, tb = run()
    for u, v, w in zip(a, t, b):
        assert np.array_equal(u, w)                 # fp32 before and after a TF32 round: bitwise equal
        assert _rel(v, u) > 1e-5                    # TF32 differs from fp32
    assert la == lt == lb and ta == tt == tb > 0    # same launches and tensor-core launches in both modes


@pytest.mark.parametrize('prec', ['fp32', 'tf32'])
def test_dilated_on_one_receptive_field_equals_optimized1f(prec):
    dil = _model(17, (3, 3, 3), 64, strided=False).cuda()
    one = _model(17, (3, 3, 3), 64, strided=True).cuda()
    one.load_state_dict(dil.state_dict())
    engine.set_precision(dil, prec)
    engine.set_precision(one, prec)
    x = torch.from_numpy(synth.synth_input(9, 27, 17, 2, seed=3)).cuda()
    with torch.no_grad():
        assert torch.equal(dil(x), one(x))


def test_mpjpe_and_profile_follow_the_setting():
    m = engine.set_precision(_model(17, (3, 3, 3), 64).cuda(), 'tf32')
    x = torch.from_numpy(synth.synth_input(4, 27, 17, 2, seed=1)).cuda()
    with torch.no_grad():
        y = m(x)
    y2, loss = engine.run_model_mpjpe(m, x, torch.zeros_like(y))
    assert torch.equal(y, y2)
    assert abs(float(loss) - float(y.double().norm(dim=-1).mean())) < 1e-5 * float(loss)
    prof = engine.profile_forward(m, x, reps=1)
    assert prof['gemm_core'].startswith('wgmma-1xtf32'), prof['gemm_core']
    engine.set_precision(m, 'fp32')
    assert engine.profile_forward(m, x, reps=1)['gemm_core'].startswith('wgmma-3xtf32')


# ------------------------------------------------------------------------------------------------------------------
# streams
# ------------------------------------------------------------------------------------------------------------------
def _seq(J, T, seed):
    return synth.synth_input(1, T, J, 2, seed=seed)[0]


@pytest.mark.parametrize('fw,ch,causal', [((3, 3, 3), 128, False), ((3, 3, 3), 64, True)])
def test_lift_sequences_equals_evaluate_sequence(fw, ch, causal):
    m = _model(17, fw, ch, causal=causal).cuda()
    lengths = [70, 5, 33, 90]
    seqs = [_seq(17, L, 100 + L) for L in lengths]
    kl, kr = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    worst = {}
    for prec in ('fp32', 'tf32'):
        engine.set_precision(m, prec)
        out = lift_sequences(m, seqs, n_streams=2, chunk=24, augment=True)
        w = 0.0
        for k, sq in enumerate(seqs):
            want = tta.evaluate_sequence(m, sq, kl, kr, kl, kr, causal=causal).cpu().numpy()
            w = max(w, _rel(out[k].cpu().numpy(), want))
        worst[prec] = w
    report('lift vs evaluate_sequence %s c%d causal %d: fp32 %.2e, tf32 %.2e' % (fw, ch, causal, worst['fp32'],
                                                                                 worst['tf32']))
    if worst['fp32'] == 0.0:
        assert worst['tf32'] == 0.0                 # bit for bit, as in fp32
    else:
        assert worst['tf32'] <= EXACT_BAR


def _stream_poses(ps, seq, pushes):
    """push `seq` (T, J, 2) on stream 0 of a 2-stream PoseStream (stream 1 gets the mirrored sequence) by `pushes`
    (list of chunk lengths, 1 = a single push), end it, flush -> poses (T, J, 3) of stream 0"""
    T = seq.shape[0]
    both = np.stack([seq, seq[::-1].copy()])
    got = {}
    t = 0
    for K in pushes + [1] * (T + ps.latency):
        if t >= T + ps.latency:
            break
        if t == T:
            ps.end()
        if t < T and K > 1:
            K = min(K, T - t)
            y, idx = ps.push_frames(torch.from_numpy(both[:, t:t + K].copy()).cuda())
            y = y.cpu().numpy()
            for k in range(K):
                if idx[0, k] >= 0:
                    got[int(idx[0, k])] = y[0, k]
        else:
            fr = both[:, min(t, T - 1)]
            y, idx = ps.push(torch.from_numpy(fr.copy()).cuda())
            if idx[0] >= 0:
                got[int(idx[0])] = y[0].cpu().numpy()
            K = 1
        t += K
    return np.stack([got[i] for i in range(T)])


def test_pose_stream_push_and_chunks_in_tf32():
    m = engine.set_precision(_model(17, (3, 3, 3), 64).cuda(), 'tf32')
    seq = _seq(17, 60, 5)
    kl, kr = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    whole = tta.evaluate_sequence(m, seq, kl, kr, kl, kr).cpu().numpy()
    ps = PoseStream(m, 2, augment=True)
    single = _stream_poses(ps, seq, [])
    launches = ps.last_launches
    ps = PoseStream(m, 2, augment=True)
    chunked = _stream_poses(ps, seq, [7, 1, 30, 2])
    e1, e2 = _l2(single, whole), _l2(chunked, whole)
    report('PoseStream augment in tf32 against the whole sequence: L2 push %.2e, chunks %.2e; max %.2e, %.2e'
           % (e1, e2, _rel(single, whole), _rel(chunked, whole)))
    assert e1 <= STREAM_L2_BAR and e2 <= STREAM_L2_BAR
    assert _rel(single, whole) < EXACT_BAR and _rel(chunked, whole) < EXACT_BAR
    engine.set_precision(m, 'fp32')
    ps = PoseStream(m, 2, augment=True)
    ref32 = _stream_poses(ps, seq, [])
    assert ps.last_launches == launches               # per-push launches do not depend on the precision
    assert _rel(single, ref32) > 1e-5                 # the streams follow the setting


def test_causal_stream_switch_mid_stream():
    m = _model(17, (3, 3, 3), 64, causal=True).cuda()
    T, rf = 50, m.receptive_field()
    seq = _seq(17, T, 9)
    padded = np.pad(seq, ((rf - 1, 0), (0, 0), (0, 0)), 'edge')[None]
    with torch.no_grad():
        exact = m(torch.from_numpy(padded).cuda())[0].cpu().numpy()          # fp32-grade whole sequence
    cs = CausalStream(m, 1)
    out = []
    for t in range(T):
        if t == T // 2:
            engine.set_precision(m, 'tf32')                                    # no weight change: no refusal
        y = cs.push(torch.from_numpy(seq[t:t + 1].copy()).cuda())
        out.append(y[0].cpu().numpy() if isinstance(y, torch.Tensor) else y[0][0].cpu().numpy())
    out = np.stack(out)
    e_first, e_second = _rel(out[:T // 2], exact[:T // 2]), _rel(out[T // 2:], exact[T // 2:])
    report('CausalStream switched to tf32 at push %d: before %.2e, after %.2e' % (T // 2, e_first, e_second))
    assert e_first < 1e-5
    assert 1e-5 < e_second < EXACT_BAR
    engine.set_precision(m, 'fp32')


# ------------------------------------------------------------------------------------------------------------------
# refusals
# ------------------------------------------------------------------------------------------------------------------
def test_refusals():
    m = engine.set_precision(_model(17, (3, 3, 3), 32).cuda(), 'tf32')
    x = torch.from_numpy(synth.synth_input(2, 27, 17, 2, seed=2)).cuda()
    m.train()
    with pytest.raises(engine.GastError, match=r"set_precision\(model, 'fp32'\)"):
        m(x)
    m.eval()
    with pytest.raises(engine.GastError, match=r"set_precision\(model, 'fp32'\)"):
        m(x.clone().requires_grad_(True))
    with pytest.raises(engine.GastError, match=r"set_precision\(model, 'fp32'\)"):
        m(x)                                          # parameters require grad and grad mode is on
    with torch.no_grad():
        m(x)                                          # inference runs
    with pytest.raises(engine.GastError):
        engine.set_precision(m, 'bf16')
    h = _handle(m)
    lib = h.lib
    assert lib.gast_set_precision(h.h, 2) != 0 and 'mode' in _lib.last_error()
    assert lib.gast_set_precision(h.h, -1) != 0
    assert lib.gast_set_precision(h.h, 1) == 0
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.gast_train_workspace_bytes(h.h, 2, 27, C.c_float(0.0)) == 0
    assert 'inference-only' in _lib.last_error()
    assert lib.gast_eval_backward_workspace_bytes(h.h, 2, 27, 1) == 0
    assert 'inference-only' in _lib.last_error()
    assert lib.gast_forward_train(h.h, None, None, 2, 27, C.c_float(0.0), C.c_uint64(0), None, 0, st) != 0
    assert 'inference-only' in _lib.last_error()
    assert lib.gast_backward(h.h, None, None, 0, st) != 0
    assert 'inference-only' in _lib.last_error()
    assert lib.gast_backward_input(h.h, None, None, 1, None, 0, st) != 0
    assert 'inference-only' in _lib.last_error()
    assert lib.gast_eval_backward(h.h, None, None, None, 1, 2, 27, 1, None, 0, st) != 0
    assert 'inference-only' in _lib.last_error()
    # back to fp32: training works again on the same module
    engine.set_precision(m, 'fp32')
    m.train()
    y = m(x)
    y.abs().mean().backward()
    assert all(p.grad is not None for p in m.parameters() if p.requires_grad)


def test_deepcopy_keeps_the_setting_on_its_own_handle():
    m = engine.set_precision(_model(17, (3, 3, 3), 64).cuda(), 'tf32')
    x = torch.from_numpy(synth.synth_input(3, 27, 17, 2, seed=4)).cuda()
    with torch.no_grad():
        y = m(x)
        c = copy.deepcopy(m)
        assert engine.get_precision(c) == 'tf32'
        assert torch.equal(c(x), y)
        assert '_gast_precision' not in ''.join(m.state_dict().keys())
