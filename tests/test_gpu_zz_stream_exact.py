"""GPU: every pose the O(1) causal stream returns (gast_b200.realtime.CausalStream, C ABI gast_stream_push) against the
fp64 per-frame reference of tests/streamref.py, on both GEMM cores, over a matrix of ring geometries, stream counts,
joint counts and widths, with resets placed on ring wraps, tile boundaries and consecutive pushes.

The matrix reaches (test_case_matrix_reaches_stream_branches checks it): every tap-rotated weight copy of every stage
(up to 5 taps, the 243-slot ring over more than two revolutions); a first filter width of 5 (expand_rows_kernel<10>
and a 5-frame input history); frame tiles of 120, 128 (exact), 119 (ragged tail) and 114 rows; several flat tiles and
the attention mix kernel's tail block; stream_fill_fresh_kernel with gridDim.y of 1, 4 and 8; a second grid-stride
pass of rowdot8_kernel; 16 channels (the first block on the FFMA core even on the default core), 48 (both cores in
one push) and 160 (a ragged second N tile of the tensor-core GEMM); step counters from 0 and from 2^40 + phase.

Measured on an H100 80GB HBM3 (400 W power limit), worst over the matrix, against fp64: max error / max |y64|
2.2e-6 on the default core and 2.6e-6 on the FFMA core, relative L2 1.6e-6 on either; against the GPU whole-sequence
forward 1.5e-6 (default) and 2.6e-6 (FFMA).  The bars are about 4x those.
"""
import os

import numpy as np
import pytest
import torch

from gast_b200 import engine
from gast_b200.realtime import CausalStream
import streamref as S

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')   # optional directory for the measured errors of these tests

MAX_BAR = 1e-5                     # max |y - y64| / max |y64|, either GEMM core
L2_BAR = 6e-6                      # relative L2 error
WHOLE_BAR = 1e-5                   # max |y - y_whole| / max |y|: push against the GPU whole-sequence forward

BIG = 2 ** 40


def phase_start(fw):
    """2^40 + phase, with phase chosen so that the first push writes the last slot of every ring (step = -1 mod
    rf = R_max, and every R_i divides rf): every stage starts on its last tap-rotated weight copy"""
    return BIG + (-1 - BIG) % S.receptive_field(fw)


Case = S.Case
CASES = {
    # 6 frame tiles (ragged tail of 2 streams), 5 flat tiles, mix tail blocks, fill-fresh gridDim.y 4 and 8.  Resets:
    # streams 6 and 7 (both sides of the first frame tile), stream 7 on two consecutive pushes, every stream, and at
    # step 27 where the 27-slot ring wraps to slot 0
    'j17_333_c128_n37': Case(17, (3, 3, 3), 128, 37, 30, 0, ((12, (6, 7)), (13, (7,)), (20, None), (27, (0, 36))), 1),
    # first width 5; 48 channels: the first block on the FFMA core (K % 32 != 0), the 96-channel stage and block on
    # tensor cores.  Starts at
    # 2^40 + phase; push 1 and push 16 land on slot 0 of the 15-slot ring
    'j15_53_c48_n9': Case(15, (5, 3), 48, 9, 20, phase_start((5, 3)), ((1, (3,)), (7, (4, 5)), (8, (5,)), (16, None)), 2),
    # a 5-tap stage (rotation copies 0..4), exact 128-row frame tiles of 8 streams; reset at the 45-slot wrap
    'j16_353_c32_n16': Case(16, (3, 5, 3), 32, 16, 50, 0, ((10, None), (30, (15,)), (31, (15,)), (45, (7, 8))), 3),
    # 16 channels: the first block on FFMA (K % 32 != 0) on either core, later stages on tensor cores; 114-row tiles.
    # Starts at 2^40 + phase: pushes 1 and 82 land on slot 0 of the 81-slot ring
    'j19_3333_c16_n7': Case(19, (3, 3, 3, 3), 16, 7, 90, phase_start((3, 3, 3, 3)),
                            ((1, (0, 6)), (40, (3,)), (41, (3,)), (82, None)), 4),
    # the 243-frame model: stream 0 runs through the 243-slot ring more than three times
    'j17_33333_c16_n3': Case(17, (3, 3, 3, 3, 3), 16, 3, 740, 0, ((243, (1,)), (300, (2,)), (301, (2,))), 5),
    # a ragged second N tile of the tensor-core GEMM (160 channels)
    'j17_333_c160_n5': Case(17, (3, 3, 3), 160, 5, 30, 0, ((27, (2,)), (28, (4,))), 6),
    # many streams: rowdot8_kernel's second grid-stride pass, 92 frame tiles, many mix blocks
    'j17_333_c32_n640': Case(17, (3, 3, 3), 32, 640, 28, 0, ((9, (0, 639)), (14, tuple(range(300, 340))), (27, None)), 7),
}

FULL_CHECK = 64     # up to this many streams every stream is compared with fp64; above it a sample (see `sample`)


def stages(case):
    """[(taps w_i, dilation d_i, ring slots R_i, ring width Cw_i)] of temporal stages 1..L-1 (csrc/stream.cuh)"""
    out, d = [], case.fw[0]
    for i in range(1, len(case.fw)):
        out.append((case.fw[i], d, case.fw[i] * d, case.ch << i))
        d *= case.fw[i]
    return out


def block_widths(case):
    return [case.ch << i for i in range(len(case.fw))]


def mix_frames_per_block(case, C):
    """frames per block of global_mix_kernel for a block of C channels (run_global in csrc/gast_api.cu)"""
    fpb = max(1, 128 // (C // 4))
    return max(1, min(fpb, 40 * 1024 // (4 * 4 * case.J * 20)))


def rowdot8_blocks_per_pass(sms):
    return 8 * sms


def sample(case, sms):
    """streams of a many-stream case that are compared with fp64: the first and the last, both sides of the first
    three and the last boundary of the frame tiles, the flat 128-row tiles, the mix blocks and rowdot8_kernel's
    grid-stride passes, and every stream that is reset"""
    n, J = case.n, case.J
    if n <= FULL_CHECK:
        return tuple(range(n))
    cuts = []
    for step_ in [128 // J] + [mix_frames_per_block(case, C) for C in block_widths(case)]:
        b = list(range(step_, n, step_))                      # first stream of each frame tile / mix block
        cuts += b[:3] + b[-1:]
    flat = [-(-128 * k // J) for k in range(1, n * J // 128 + 1)]     # first stream wholly past row 128 k
    cuts += flat[:3] + flat[-1:]
    cuts += [-(-rowdot8_blocks_per_pass(sms) * 8 * k // J) for k in (1, 2)]   # 8 rows per block of 256 threads
    s = {0, n - 1}
    for c in cuts:
        s.update((c - 1, c))
    for _, ss in case.resets:
        s.update(range(n) if ss is None else ss)
    if len(s) > n // 2:                                       # a reset of every stream: keep the boundaries only
        s = {0, n - 1} | {c - 1 for c in cuts} | set(cuts)
        for _, ss in case.resets:
            s.update(ss or ())
    return tuple(sorted(t for t in s if 0 <= t < n))


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def push_all(case, model, between=None, core_at=None):
    """push every frame of `case` through a CausalStream on `model` with the case's resets and step counter ->
    (n, T, J, 3) numpy.  between(t): called after push t; core_at {t: core}: set_gemm_core before push t"""
    x = torch.from_numpy(S.frames(case)).cuda()
    cs = CausalStream(model, case.n)
    cs.step = case.start
    resets = {}
    for t, ss in case.resets:
        resets.setdefault(t, []).append(ss)
    out = []
    for t in range(case.T):
        if core_at and t in core_at:
            engine.set_gemm_core(core_at[t])
        for ss in resets.get(t, []):
            cs.reset(None if ss is None else list(ss))
        out.append(cs.push(x[t]))
        if between is not None:
            between(t)
    return torch.stack(out, dim=1).cpu().numpy()


def whole_sequence(case):
    """the GPU whole-sequence forward of the dilated causal model on every padded segment -> (n, T, J, 3)"""
    m = S.module(case, dilated=True).cuda()
    rf = S.receptive_field(case.fw)
    x = S.frames(case)
    y = np.zeros((case.n, case.T, case.J, 3), dtype=np.float32)
    groups = {}
    for s in range(case.n):
        for t0, t1 in S.segments(case, s):
            groups.setdefault(t1 - t0, []).append((s, t0, t1))
    with torch.no_grad():
        for _, segs in sorted(groups.items()):
            xs = np.stack([S.padded(x[t0:t1, s], rf) for s, t0, t1 in segs])
            got = m(torch.from_numpy(xs).cuda()).cpu().numpy()
            for (s, t0, t1), g in zip(segs, got):
                y[s, t0:t1] = g
    return y


def report(line):
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        with open(os.path.join(REPORT_DIR, 'stream_exact.txt'), 'a') as f:
            f.write(line + '\n')


def test_case_matrix_reaches_stream_branches():
    """the matrix reaches what the module docstring claims, for this device's SM count"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gridy, exact, ragged, second_pass, wraps, twice, every = set(), False, False, False, 0, 0, 0
    for name, c in CASES.items():
        rf = S.receptive_field(c.fw)
        for w, d, R, Cw in stages(c):
            used = {((c.start + t) % R) // d for t in range(c.T)}
            assert used == set(range(w)), (name, w, d, used)                       # every rotation copy
            gridy.add(max(1, min(8, c.J * Cw // 4 // 256)))                        # stream_fill_fresh_kernel
        fpt = 128 // c.J
        exact |= c.n % fpt == 0
        ragged |= c.n % fpt != 0
        second_pass |= any(C % 4 == 0 and (c.n * c.J * 32 + 255) // 256 > rowdot8_blocks_per_pass(sms)
                           for C in block_widths(c))
        wraps += any(t > 0 and (c.start + t) % rf == 0 for t, _ in c.resets)
        twice += any(ss and any(t + 1 == t2 and set(ss) & set(ss2 or range(c.n)) for t2, ss2 in c.resets)
                     for t, ss in c.resets)                                    # one stream on consecutive pushes
        every += any(ss is None for _, ss in c.resets)
    assert 1 in gridy and 8 in gridy and any(1 < g < 8 for g in gridy), gridy
    assert exact and ragged
    assert second_pass
    assert wraps >= 4 and twice >= 3 and every >= 3, (wraps, twice, every)
    assert {5} <= {c.fw[0] for c in CASES.values()} and any(5 in c.fw[1:] for c in CASES.values())
    assert max(c.T - 1 for c in CASES.values() if S.receptive_field(c.fw) == 243) > 2 * 243
    assert {c.J for c in CASES.values()} == {15, 16, 17, 19}
    assert any(c.start >= BIG for c in CASES.values())
    # the first block on FFMA (K % 32 != 0), and a case whose blocks and stages land on different cores
    assert any(c.ch % 32 for c in CASES.values()) and 48 in {c.ch for c in CASES.values()}
    assert 160 in {c.ch for c in CASES.values()}


@pytest.mark.parametrize('name', sorted(CASES))
def test_stream_vs_fp64(name, core):
    case = CASES[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got = push_all(case, S.module(case).cuda())
    picked = sample(case, sms)
    mx, l2 = S.errors(got[list(picked)], S.reference(case, picked))
    whole = whole_sequence(case)
    w = float(np.abs(got - whole).max() / np.abs(whole).max())
    report('%s core %d: max %.2e l2 %.2e | vs whole-sequence %.2e | %d of %d streams vs fp64'
           % (name, core, mx, l2, w, len(picked), case.n))
    assert mx <= MAX_BAR and l2 <= L2_BAR, (mx, l2)
    assert w <= WHOLE_BAR, w


def test_gemm_core_switch_mid_stream():
    """switching the GEMM core between pushes keeps the streams (no error) and the poses within the bars"""
    case = CASES['j15_53_c48_n9']
    try:
        got = push_all(case, S.module(case).cuda(), core_at={0: 0, 6: 1, 13: 0})
    finally:
        engine.set_gemm_core(0)
    mx, l2 = S.errors(got, S.reference(case))
    report('core switch %s: max %.2e l2 %.2e' % ('j15_53_c48_n9', mx, l2))
    assert mx <= MAX_BAR and l2 <= L2_BAR, (mx, l2)


def test_dilated_handle_streams_bitwise_like_optimized1f(core):
    """SpatioTemporalModel(causal=True) with the same weights folds to the same constants and runs the same launches"""
    case = CASES['j16_353_c32_n16']
    a = push_all(case, S.module(case).cuda())
    b = push_all(case, S.module(case, dilated=True).cuda())
    assert np.array_equal(a, b), float(np.abs(a - b).max())


def test_pushes_isolated_from_forwards_and_eval_backward_on_the_same_model():
    """eval forwards of other batches and an eval backward on the same model between pushes change no pushed bit"""
    case = CASES['j17_333_c128_n37']
    plain = push_all(case, S.module(case).cuda())
    m = S.module(case).cuda()
    rf = S.receptive_field(case.fw)
    other = torch.from_numpy(np.random.RandomState(9).uniform(-1, 1, (5, rf, case.J, 2)).astype(np.float32)).cuda()

    def between(t):
        if t % 3 == 0:
            with torch.no_grad():
                m(other[: 1 + t % 5])
        if t % 7 == 3:
            xg = other.clone().requires_grad_()
            m(xg).square().sum().backward()
            assert xg.grad is not None
    mixed = push_all(case, m, between=between)
    assert np.array_equal(plain, mixed), float(np.abs(plain - mixed).max())


WEIGHT_CASE = Case(17, (3, 3, 3), 32, 4, 14, 0, (), 11)


def _change(kind, m, case):
    if kind == 'load_state_dict':
        m.load_state_dict(S.module(case._replace(seed=case.seed + 1)).state_dict())
    elif kind == 'optimiser_step':
        opt = torch.optim.SGD(m.parameters(), lr=1e-2)
        for p in m.parameters():
            p.grad = torch.full_like(p, 0.1)
        opt.step()
    else:                                       # one training step: moves the BatchNorm running statistics
        m.train()
        x = torch.from_numpy(np.random.RandomState(3).uniform(-1, 1, (4, 27, case.J, 2)).astype(np.float32)).cuda()
        m(x).square().mean().backward()
        m.eval()
        m.zero_grad(set_to_none=True)


@pytest.mark.parametrize('kind', ['load_state_dict', 'optimiser_step', 'training_step'])
def test_weight_change_under_live_stream_raises_until_reset(kind):
    case = WEIGHT_CASE
    m = S.module(case).cuda()
    x = torch.from_numpy(S.frames(case)).cuda()
    cs = CausalStream(m, case.n)
    t0 = 6
    for t in range(t0):
        cs.push(x[t])
    engine.set_gemm_core(1)                     # a core switch is not a weight change
    try:
        cs.push(x[t0])
    finally:
        engine.set_gemm_core(0)
    t0 += 1
    _change(kind, m, case)
    with pytest.raises(engine.GastError, match='reset'):
        cs.push(x[t0])
    cs.reset([0, 1])                            # some streams keep their old-weight history: still refused
    with pytest.raises(engine.GastError, match='reset'):
        cs.push(x[t0])
    cs.reset()
    got = torch.stack([cs.push(x[t]) for t in range(t0, case.T)], dim=1).cpu().numpy()
    # the reference of the new weights, every stream restarting at t0
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    ref_case = case._replace(resets=((t0, None),))
    ref = S.poses(ref_case, S.frames(case), tuple(range(case.n)), state_dict=sd)[:, t0:]
    mx, l2 = S.errors(got, ref)
    assert mx <= MAX_BAR and l2 <= L2_BAR, (mx, l2)
