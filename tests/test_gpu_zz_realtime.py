"""GPU: frame-by-frame causal lifting (gast_b200.realtime.CausalStream, SURVEY.md 8f N4) equals the whole-sequence
causal forward the reference would run (UnchunkedGenerator(pad, causal_shift=pad) + dilated SpatioTemporalModel,
main.py:299-320).  Runs last: it only composes kernels the other GPU tests have already checked."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from gast_b200 import synth
from gast_b200.realtime import CausalStream, WindowStream
from test_gpu_parity import build_model

pytestmark = pytest.mark.gpu

# Absolute bars, about 4x the worst over both GEMM cores measured on an H100 80GB HBM3 (400 W power limit): stream
# against the whole-sequence forward 1.0e-6, against the stream_* goldens 5.0e-6 (the goldens' own fp32 rounding is
# about 2e-6 of max |y|, tests/test_streamref_cpu.py), O(1) rings against window recomputation 3.6e-6 (max |y| 3.1).
# tests/test_gpu_zz_stream_exact.py holds every push to fp64.
WHOLE_TOL = 5e-6
GOLDEN_TOL = 2e-5
WINDOW_TOL = 1.5e-5


def test_causal_stream_equals_full_sequence_forward():
    g1f = load_golden('model_17_333_c16_causal_1f_T27')          # causal Optimized1f, as gen_skes.load_model_realtime builds
    gfull = load_golden('model_17_333_c16_causal_full_T30')      # the same network as a dilated causal SpatioTemporalModel
    m1f = build_model(g1f['meta'])
    mfull = build_model(gfull['meta'])
    mfull.load_state_dict(m1f.state_dict())                      # identical key lists (main.py:252 relies on it)
    rf = m1f.receptive_field()
    T, n = 40, 3
    seqs = np.stack([synth.synth_input(1, T, 17, 2, seed=50 + s)[0] for s in range(n)])      # (n, T, 17, 2)
    cs = CausalStream(m1f, n_streams=n)
    got = torch.stack([cs.push(torch.from_numpy(seqs[:, t]).cuda()) for t in range(T)], dim=1)   # (n, T, 17, 3)
    padded = np.pad(seqs, ((0, 0), (rf - 1, 0), (0, 0), (0, 0)), 'edge')                      # pad + causal_shift on the left
    with torch.no_grad():
        want = mfull(torch.from_numpy(padded).cuda())
    assert want.shape == got.shape == (n, T, 17, 3)
    assert (got - want).abs().max().item() < WHOLE_TOL


@pytest.mark.parametrize('name', ['stream_17_333_c32_causal', 'stream_17_333_c128_causal', 'stream_17_3333_c64_causal'])
def test_causal_stream_vs_reference_golden(name):
    """frame-by-frame output against what the UNMODIFIED reference produced for every frame of the sequence
    (its UnchunkedGenerator(pad, causal_shift=pad) + causal model, tests/golden/make_golden.py:stream_cases)"""
    from model.gast_net import SpatioTemporalModelOptimized1f
    from test_gpu_parity import _adj
    g = load_golden(name)
    meta = g['meta']
    m = SpatioTemporalModelOptimized1f(_adj(17), 17, 2, 17, meta['filter_widths'], causal=True, dropout=0.05,
                                       channels=meta['channels'])
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == meta['keys']
    synth.randomize_module(m, meta['seed'])
    m = m.cuda().eval()
    x, y = g['x'], g['y']                                         # (n, T, 17, 2), (n, T, 17, 3)
    cs = CausalStream(m, n_streams=x.shape[0])
    got = torch.stack([cs.push(torch.from_numpy(x[:, t]).cuda()) for t in range(x.shape[1])], dim=1).cpu().numpy()
    err = float(np.abs(got - y).max())
    assert err < GOLDEN_TOL, err
    # a stream that restarts: same outputs again
    cs.reset()
    again = torch.stack([cs.push(torch.from_numpy(x[:, t]).cuda()) for t in range(5)], dim=1).cpu().numpy()
    assert np.abs(again - y[:, :5]).max() < GOLDEN_TOL


def test_o1_stream_matches_window_recompute_with_staggered_resets():
    """the O(1) rings (CausalStream) against the recompute-the-window driver (WindowStream) on the same causal
    network, with streams that restart at different times, wider than one ring revolution (81-frame model:
    rings of 9, 27 and 81 slots)"""
    from model.gast_net import SpatioTemporalModelOptimized1f
    from test_gpu_parity import _adj
    m = SpatioTemporalModelOptimized1f(_adj(17), 17, 2, 17, [3, 3, 3, 3], causal=True, dropout=0.05, channels=32)
    synth.randomize_module(m, 12)
    m = m.cuda().eval()
    n, T = 5, 100
    seqs = torch.from_numpy(synth.synth_input(n, T, 17, 2, seed=31)).cuda()
    a, b = CausalStream(m, n), WindowStream(m, n)
    assert a.push(seqs[:, 0]).shape == (n, 17, 3)
    a.reset(); b_out = None
    worst = 0.0
    for t in range(T):
        if t == 37:
            a.reset([1, 3]); b.reset([1, 3])
        if t == 90:
            a.reset([0]); b.reset([0])
        ya, yb = a.push(seqs[:, t]), b.push(seqs[:, t])
        worst = max(worst, (ya - yb).abs().max().item())
    assert worst < WINDOW_TOL, worst
    assert a.last_launches < 60                       # one position per layer: ~40 launches per frame, any n
    with pytest.raises(RuntimeError, match='causal'):
        CausalStream(SpatioTemporalModelOptimized1f(_adj(17), 17, 2, 17, [3, 3, 3], channels=32).cuda().eval(), 2)
