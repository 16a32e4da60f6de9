"""GPU parity: the CUDA path (through the C ABI, via the drop-in modules) against
(i) golden outputs of the unmodified reference and (ii) the numpy oracle on seeded inputs.
Tolerance: 1e-4 absolute per coordinate in fp32 (BASELINE.json north_star); the FFMA core
is held to 2e-5."""
import numpy as np
import pytest
import torch

from conftest import load_golden, golden_names
from gast_b200 import synth, engine

pytestmark = pytest.mark.gpu

TOL = 1e-4
TOL_FFMA = 2e-5


def _adj(J):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))


def build_model(meta, device='cuda'):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    J = meta['J']
    if meta['strided']:
        m = SpatioTemporalModelOptimized1f(_adj(J), J, 2, J, meta['filter_widths'], causal=meta['causal'],
                                           dropout=0.05, channels=meta['channels'])
    else:
        m = SpatioTemporalModel(_adj(J), J, 2, J, meta['filter_widths'], causal=meta['causal'],
                                dropout=0.05, channels=meta['channels'], dense=meta['dense'])
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == meta['keys']
    synth.randomize_module(m, meta['seed'])
    return m.to(device).eval()


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def tc_launches(m):
    """kernels of the last forward that ran on the tensor-core GEMM core"""
    h = list(m.__dict__['_gast_handles'].values())[0]
    return int(h.lib.gast_last_tc_launch_count(h.h))


@pytest.mark.parametrize('name', golden_names('model_') + golden_names('cfg') + golden_names('tc_'))
def test_model_vs_reference_golden(name, core):
    g = load_golden(name)
    m = build_model(g['meta'])
    with torch.no_grad():
        y = m(torch.from_numpy(g['x']).cuda())
    assert tuple(y.shape) == g['y'].shape
    err = np.abs(y.cpu().numpy() - g['y']).max()
    assert err < (TOL_FFMA if core == 1 else TOL), err
    if name.startswith('tc_') or name.startswith('cfg'):
        # widths that are multiples of 32: every skeleton / geometry of these goldens is seen by the tensor-core
        # kernels (J = 15, 16, 17, 19; 2-5 stages; dense; causal; dilated long-sequence mode), not by the FFMA twin
        assert (tc_launches(m) > 0) == (core == 0)
    assert m.receptive_field() == g['meta']['receptive_field']
    assert m.total_causal_shift() == g['meta']['total_causal_shift']
    assert m.pad == g['meta']['pad'] and m.causal_shift == g['meta']['causal_shift']


def test_modules_vs_reference_golden(core):
    from model.gast_net import GraphAttentionBlock
    from model.local_attention import LocalGraph, SemCHGraphConv, local_adjacencies
    from model.global_attention import MultiGlobalGraph, GlobalGraph
    from model.sem_graph_conv import SemGraphConv
    tol = TOL_FFMA if core == 1 else TOL
    for name in ('mod_block_17_32', 'mod_block_19_16'):
        g = load_golden(name)
        J, Cc = g['meta']['J'], g['meta']['C']
        blk = GraphAttentionBlock(_adj(J), Cc, Cc, 0.05)
        synth.randomize_module(blk, g['meta']['seed'])
        blk = blk.cuda().eval()
        y = blk(torch.from_numpy(g['x']).cuda().permute(0, 3, 1, 2))
        assert np.abs(y.cpu().numpy() - g['y']).max() < tol
    g = load_golden('mod_local_17_32')
    lg = LocalGraph(_adj(17), 32, 32, 0.05)
    synth.randomize_module(lg, g['meta']['seed'])
    y = lg.cuda().eval()(torch.from_numpy(g['x']).cuda())
    assert np.abs(y.cpu().numpy() - g['y']).max() < tol
    g = load_golden('mod_mglobal_17_32')
    mg = MultiGlobalGraph(_adj(17), 32, 8, dropout=0.05)
    synth.randomize_module(mg, g['meta']['seed'])
    y = mg.cuda().eval()(torch.from_numpy(g['x']).cuda())
    assert np.abs(y.cpu().numpy() - g['y']).max() < tol
    g = load_golden('mod_global_17_32')
    gg = GlobalGraph(_adj(17), 32, 8)
    synth.randomize_module(gg, g['meta']['seed'])
    y = gg.cuda().eval()(torch.from_numpy(g['x']).cuda())
    assert np.abs(y.cpu().numpy() - g['y']).max() < tol
    _, con = local_adjacencies(_adj(17))
    g = load_golden('mod_semch_17_32')
    sc = SemCHGraphConv(32, 32, con)
    synth.randomize_module(sc, g['meta']['seed'])
    y = sc.cuda()(torch.from_numpy(g['x']).cuda())
    assert np.abs(y.cpu().numpy() - g['y']).max() < tol
    g = load_golden('mod_semgc_17_32')
    sg = SemGraphConv(32, 32, con, bias=True)
    synth.randomize_module(sg, g['meta']['seed'])
    y = sg.cuda()(torch.from_numpy(g['x']).cuda())
    assert np.abs(y.cpu().numpy() - g['y']).max() < tol


def test_against_oracle_random_shapes(core):
    """seeded inputs at sizes the numpy oracle finishes in seconds; odd batch / ragged tiles."""
    from oracle import gast_oracle as O
    tol = TOL_FFMA if core == 1 else TOL
    for (J, fw, ch, B, T, strided, causal) in [
            (17, [3, 3, 3], 32, 5, 27, True, False),
            (17, [3, 3, 3], 32, 1, 33, False, False),
            (19, [3, 3], 32, 3, 11, False, True),
            (15, [3, 3, 3], 16, 2, 27, True, True),
            (17, [3, 3, 3], 64, 9, 27, False, False),
            (17, [3, 3], 1056, 3, 9, True, False)]:        # > 1024 channels: two channel chunks in the expand
        meta = dict(J=J, filter_widths=fw, channels=ch, strided=strided, causal=causal, dense=False, seed=11)
        from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
        cls = SpatioTemporalModelOptimized1f if strided else SpatioTemporalModel
        m = cls(_adj(J), J, 2, J, fw, causal=causal, dropout=0.05, channels=ch)
        synth.randomize_module(m, 11)
        p = {k: v.numpy() for k, v in m.state_dict().items()}
        x = synth.synth_input(B, T, J, 2, seed=99 + B)
        ref = O.forward(x, p, O.adj_from_parents(synth.skeleton_parents(J)), fw, causal=causal, strided=strided)
        with torch.no_grad():
            y = m.cuda().eval()(torch.from_numpy(x).cuda()).cpu().numpy()
        assert y.shape == ref.shape
        assert np.abs(y - ref).max() < tol, (J, fw, ch, B, T, np.abs(y - ref).max())


def test_tc_gemm_accuracy_at_any_weight_scale():
    """The tensor-core GEMM core (3xTF32, csrc/gemm_tc.cuh) keeps fp32's range and fp32-grade error: one GEMM through
    gast_debug_gemm (core 0) against fp64, with ordinary weights and with weights far outside fp16's range."""
    import ctypes as C
    from gast_b200 import _lib
    lib = _lib.load()
    rs = np.random.RandomState(3)
    M, N, K = 384, 128, 512
    A = rs.standard_normal((M, K)).astype(np.float32)
    for wscale, bar in ((1.0 / np.sqrt(K), 2e-6), (300.0, 2e-6)):          # second: 2^8 * max|W| ~ 3e5 > 65504
        W = (rs.standard_normal((N, K)) * wscale).astype(np.float32)
        a, w = torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda()
        o = torch.empty((M, N), dtype=torch.float32, device='cuda')
        rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, 0, 0, None,
                                 torch.cuda.current_stream().cuda_stream)
        assert rc == 0, _lib.last_error()
        ref = A.astype(np.float64) @ W.astype(np.float64).T
        d = o.cpu().numpy().astype(np.float64) - ref
        rel = np.sqrt((d ** 2).mean()) / np.sqrt((ref ** 2).mean())
        assert np.isfinite(d).all() and rel < bar, (wscale, rel)


def test_full_size_properties():
    """BASELINE config 2 at full size (4096 clips): size-independent properties.
    (a) batch independence: a clip's output does not depend on its batch neighbours (bit-exact);
    (b) full model == Optimized1f on the same weights (state_dict interchangeable);
    (c) sliding window: T=40 sequence == 14 independent 27-frame clips;
    (d) MPJPE equal to 3 decimals (mm) between (b)'s two paths."""
    g = load_golden('cfg2_17_333_c128_full_T27')
    m = build_model(g['meta'])
    B = 4096
    x = torch.from_numpy(synth.synth_input(B, 27, 17, 2, seed=1234)).cuda()
    with torch.no_grad():
        y = m(x)
        y_head = m(x[:100].contiguous())
        assert torch.equal(y[:100], y_head)
        y_tail = m(x[B - 37:].contiguous())
        assert torch.equal(y[B - 37:], y_tail)
        meta1 = dict(g['meta'], strided=True)
        m1 = build_model(meta1)
        m1.load_state_dict(m.state_dict())
        y1 = m1(x)
        assert (y - y1).abs().max().item() < 1e-5
        # the first 4 clips of this seed are the golden's input
        assert np.abs(y[:4].cpu().numpy() - g['y']).max() < TOL
        xs = torch.from_numpy(synth.synth_input(3, 40, 17, 2, seed=5)).cuda()
        ys = m(xs)
        assert ys.shape == (3, 14, 17, 3)
        wins = torch.stack([xs[:, t:t + 27] for t in range(14)], 1).reshape(3 * 14, 27, 17, 2).contiguous()
        yw = m(wins).reshape(3, 14, 17, 3)
        assert (ys - yw).abs().max().item() < 2e-5
    gt = torch.from_numpy(synth.synth_target(B, 17)).cuda()
    mp = lambda a: (torch.norm(a - gt, dim=3).mean().item() * 1000.0)
    assert abs(mp(y) - mp(y1)) <= 5e-6 * mp(y), (mp(y), mp(y1))


@pytest.mark.parametrize('name', ['cfg2_17_333_c128_full_T27', 'cfg4_17_3333_c64_1f_T81', 'cfg5_19_333_c128_full_T27'])
def test_mpjpe_three_decimals_at_realistic_scale(name):
    """"MPJPE identical to 3 decimals" (BASELINE north_star), literally, at the scale of real poses: the output
    layer (shrink, no bias: the output is linear in its weight) is scaled by 2^-2 -- an exact operation in fp32,
    so the reference's output for the scaled weights is exactly 0.25 x its golden output -- and the ground truth
    is that output plus ~50 mm of error per joint.  MPJPE in millimetres must then agree to 3 decimals."""
    g = load_golden(name)
    m = build_model(g['meta'])
    with torch.no_grad():
        m.shrink.weight.mul_(0.25)
        y = m(torch.from_numpy(g['x']).cuda()).cpu().numpy().astype(np.float64)
    ref = 0.25 * g['y'].astype(np.float32)
    assert np.array_equal(ref, (0.25 * g['y'].astype(np.float64)).astype(np.float32))      # exact scaling
    rs = np.random.RandomState(7)
    gt = ref.astype(np.float64) + 0.031 * rs.standard_normal(ref.shape)                    # mean joint error ~50 mm
    mp = lambda a: float(np.mean(np.linalg.norm(a - gt, axis=-1)) * 1000.0)
    a, b = mp(y), mp(ref.astype(np.float64))
    assert 30.0 < b < 80.0
    assert '%.3f' % a == '%.3f' % b or abs(a - b) < 5e-4, (a, b)


def test_error_behaviour():
    from model.gast_net import SpatioTemporalModel
    from model.local_attention import LocalGraph
    m = SpatioTemporalModel(_adj(17), 17, 2, 17, [3, 3, 3], channels=16).cuda().eval()
    with pytest.raises(AssertionError):
        m(torch.zeros(2, 27, 16, 2, device='cuda'))      # gast_net.py:94
    with pytest.raises(AssertionError):
        m(torch.zeros(2, 27, 17, 3, device='cuda'))      # gast_net.py:95
    with pytest.raises(AssertionError):
        m(torch.zeros(27, 17, 2, device='cuda'))         # gast_net.py:93
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 20, 17, 2, device='cuda'))      # shorter than the receptive field
    with pytest.raises(RuntimeError):
        m(torch.zeros(2, 27, 17, 2))                     # CPU tensor: no fallback
    with pytest.raises(RuntimeError):
        m(torch.zeros(0, 27, 17, 2, device='cuda'))      # empty batch: the reference raises too (view(0, C, -1) of 0 elements, global_attention.py:56)
    with pytest.raises(KeyError):
        LocalGraph(torch.eye(14), 16, 16)                # local_attention.py:89-90
    with pytest.raises(AssertionError):
        SpatioTemporalModel(_adj(17), 17, 2, 17, [3, 4, 3], channels=16)   # gast_net.py:46-47


def test_state_dict_roundtrip_and_inplace_output():
    """load_state_dict after the first forward must be seen (main.py:252), and callers write
    into the returned tensor in place (reconstruction.py:165-166)."""
    g = load_golden('model_17_333_c16_full_T31')
    m = build_model(g['meta'])
    x = torch.from_numpy(g['x']).cuda()
    with torch.no_grad():
        y0 = m(x).clone()
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        synth.randomize_module(m, 77)
        y1 = m(x)
        assert (y1 - y0).abs().max().item() > 1e-3
        m.load_state_dict(sd)
        y2 = m(x)
        assert torch.equal(y2, y0)
        y2[1, :, :, 0] *= -1
        y2[1, :, [4, 5, 6, 1, 2, 3]] = y2[1, :, [1, 2, 3, 4, 5, 6]]
        assert torch.mean(y2, dim=0, keepdim=True).shape == (1, 5, 17, 3)


@pytest.mark.parametrize('J,fw,ch,B,T', [(17, [3, 3, 3], 128, 96, 27),        # BASELINE configs[1]/[2] shape
                                         (17, [3, 3, 3, 3], 64, 40, 81),      # configs[3]: 81-frame model
                                         (19, [3, 3, 3], 128, 75, 27),        # configs[4]: body+toe skeleton
                                         (17, [3, 3, 3], 128, 3, 60)])        # whole-sequence (dilated) mode
def test_baseline_configs_vs_torch_port(J, fw, ch, B, T, core):
    """BASELINE.json configurations at full width against the torch-CPU port of the reference
    (bit-identical to the reference modules), ragged batch sizes."""
    from oracle import gast_torch_ref as TR
    from oracle import gast_oracle as O
    from model.gast_net import SpatioTemporalModel
    m = SpatioTemporalModel(_adj(J), J, 2, J, fw, dropout=0.05, channels=ch)
    synth.randomize_module(m, 21)
    p = {k: v.clone() for k, v in m.state_dict().items()}
    masks = tuple(torch.from_numpy(a) for a in O.local_masks(O.adj_from_parents(synth.skeleton_parents(J))))
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=77))
    n_ref = min(B, 24)
    with torch.no_grad():
        rf = 1 + 2 * sum(O.model_geometry(fw, False, False)[0])
        ref = TR.forward(x[:n_ref], p, masks, fw, strided=(T == rf)).numpy()
        y = m.cuda().eval()(x.cuda()).cpu().numpy()
    assert y.shape[0] == B and y.shape[1:] == ref.shape[1:]
    err = np.abs(y[:n_ref] - ref).max()
    assert err < (TOL_FFMA if core == 1 else TOL), err
    # MPJPE (common/loss.py:5-11) against a synthetic ground truth.  The contract's "identical to 3 decimals" is
    # asserted literally at the scale of real poses in test_mpjpe_three_decimals_at_realistic_scale; the untrained
    # synthetic network here is ~2000 mm off its random target, so this check is on the RELATIVE agreement of the
    # metric: 5e-6 (= 0.00025 mm at a 50 mm MPJPE)
    gt = synth.synth_target(n_ref, J)[:, :, :, :] * np.ones((1, ref.shape[1], 1, 1), np.float32)
    mp = lambda a: float(np.mean(np.linalg.norm(a.astype(np.float64) - gt, axis=-1)) * 1000.0)
    a, b = mp(y[:n_ref]), mp(ref)
    assert abs(a - b) <= 5e-6 * b, (a, b)


def test_tta_on_device_matches_reference_generator():
    """N1: edge padding + mirrored twin and un-flip/average on the device, bit-exact against what the
    reference's UnchunkedGenerator / main.py:314-318 produced (golden tta_17), then the whole
    evaluate_sequence on the real baseball clip of reconstruction.py."""
    from oracle import gast_oracle as O
    from gast_b200 import tta
    left, right = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
    t = load_golden('tta_17')
    seq = torch.from_numpy(t['seq']).cuda()
    for name, pad, shift in (('sym', 13, 0), ('causal', 13, 13), ('pad40', 40, 0)):
        got = tta.tta_prepare(seq, pad, shift, left, right).cpu().numpy()
        assert np.array_equal(got, t['batch_' + name]), name
    merged = tta.tta_merge(torch.from_numpy(t['pred']).cuda(), left, right).cpu().numpy()
    assert np.array_equal(merged, t['merged'][0])
    with pytest.raises(RuntimeError):
        tta.tta_prepare(seq, 13, 0, [40], [1])
    g = load_golden('cfg1_baseball_17_333_c128')
    clip = g['x'][0, 13:-13]                                  # the un-padded keypoints
    assert np.array_equal(tta.tta_prepare(torch.from_numpy(clip).cuda(), 13, 0, left, right).cpu().numpy(), g['x'])
    m = build_model(g['meta'])
    out = tta.evaluate_sequence(m, clip, left, right, left, right)
    assert out.shape == (277, 17, 3)
    assert np.abs(out.cpu().numpy() - O.tta_merge(g['y'], left, right)).max() < TOL


def test_pipelined_lifter_matches_direct_calls():
    """Host-fed streaming API (gast_b200/stream.py): same poses as one direct call per batch, in order, with the
    uploads / downloads on a copy stream."""
    from gast_b200.stream import PipelinedLifter
    g = load_golden('cfg2_17_333_c128_full_T27')
    m = build_model(g['meta'])
    xs = [torch.from_numpy(synth.synth_input(64, 27, 17, 2, seed=100 + i)).pin_memory() for i in range(5)]
    outs = [torch.empty((64, 1, 17, 3), dtype=torch.float32).pin_memory() for _ in range(5)]
    PipelinedLifter(m, depth=2).run(xs, outs)
    torch.cuda.synchronize()
    with torch.no_grad():
        for x, o in zip(xs, outs):
            ref = m(x.cuda()).cpu()
            assert torch.equal(ref, o)
    with pytest.raises(RuntimeError):
        PipelinedLifter(build_model(g['meta'], device='cpu'))
