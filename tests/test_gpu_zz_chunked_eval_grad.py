"""The chunked eval-mode forward and backward (gast_forward_chunked, gast_eval_backward_chunked,
engine.run_model_chunked) on the GPU, on both GEMM cores:
  * the forward is bitwise model(x) (dilated, causal, 19 joints, the 81-frame / 64-channel model, strided with
    T > receptive field);
  * one pass is bitwise gast_eval_backward, for every parameter gradient and dL/dx, and asks for the same workspace;
  * several passes (windows that do not divide T_out, windows of one frame, whole-clip passes) agree with the
    unchunked call up to summation order, meet the rounding-level bars against the fp64 port at kink-free points
    (tests/kinkfree.py), and repeat bit for bit;
  "bitwise" and "bit for bit" hold where gast_eval_backward itself repeats bit for bit: on the strided schedule
  (Optimized1f, or a dilated model fed one receptive field).  On the dilated and dense schedules the taps of a
  temporal conv overlap, and the backward adds them into dL/d(input) with float atomics (seg_scatter_add_kernel), so
  there the unchunked call already varies in the last bits from run to run, and so does the chunked one;
  * TF32 training precision, input-only gradients, accumulation into an existing .grad, torch's in-place version
    check, the train-mode refusal, refused library calls leaving every buffer untouched, and the workspace query;
  * a recording whose unchunked eval-backward workspace exceeds device memory completes chunked, in the memory the
    chunked query promises."""
import ctypes as C
import functools

import pytest
import torch

from gast_b200 import engine, synth
import kinkfree as K

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def _mpjpe(y, t):
    return torch.mean(torch.norm(y - t, dim=3))


def _handle(m):
    return list(m.__dict__['_gast_handles'].values())[0]


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else None)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _model(J, fw, ch, strided=False, causal=False, seed=5):
    return K.module(K.Case(J, fw, ch, 1, 1, strided, causal, False, False), seed=seed).cuda().eval()


def _grads(m, x):
    g = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    if x.grad is not None:
        g['x'] = x.grad.detach().clone()
    return g


def _run(m, x, dy, max_frames=None):
    """y and every gradient of (y * dy).sum(), through model(x) (max_frames None) or run_model_chunked"""
    m.zero_grad(set_to_none=True)
    xx = x.clone().requires_grad_()
    y = m(xx) if max_frames is None else engine.run_model_chunked(m, xx, max_frames)
    y.backward(dy)
    return y.detach(), _grads(m, xx)


def _assert_bitwise(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


def _assert_same(a, b, exact):
    """bitwise when `exact`, else within the run-to-run spread of the float-atomic tap adjoints"""
    if exact:
        return _assert_bitwise(a, b)
    assert a.keys() == b.keys()
    top = max(v.abs().max().item() for v in b.values())
    for k in a:
        d = (a[k] - b[k]).abs().max().item()
        assert d <= 1e-4 * b[k].abs().max().item() + 1e-6 * top, (k, d)


# ---------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------
FORWARD_CASES = [  # J, fw, ch, strided, causal, B, T
    (17, [3, 3, 3], 32, False, False, 2, 60),
    (17, [3, 3, 3], 32, False, True, 2, 60),
    (19, [3, 3, 3], 32, False, False, 3, 40),
    (17, [3, 3, 3, 3], 64, False, False, 2, 120),
    (17, [3, 3, 3], 32, True, False, 3, 100),       # strided, T > receptive field: 3 outputs per clip
    (17, [3, 3, 3], 32, False, False, 5, 27),       # dilated at T == receptive field: the strided schedule
]


@pytest.mark.parametrize('J,fw,ch,strided,causal,B,T', FORWARD_CASES,
                         ids=['dilated', 'causal', 'j19', '81f_c64', 'strided_T100', 'dilated_rf'])
def test_forward_is_bitwise_model(J, fw, ch, strided, causal, B, T, core):
    m = _model(J, fw, ch, strided, causal)
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=1)).cuda()
    with torch.no_grad():
        y0 = m(x)
        T_out = y0.shape[1]
        for mf in sorted({1, 2, 5, T_out, T_out + 1, 2 * T_out + 1, B * T_out}):
            y = engine.run_model_chunked(m, x, mf)
            assert torch.equal(y, y0), mf
    y = engine.run_model_chunked(m, x, 3)           # the parameters require grad: the output has a backward
    assert y.grad_fn is not None and torch.equal(y, y0)
    m.requires_grad_(False)
    y = engine.run_model_chunked(m, x, 3)           # nothing requires grad: the forward alone
    assert y.grad_fn is None and torch.equal(y, y0)


# ---------------------------------------------------------------------------------------------------------------
# one pass: bitwise gast_eval_backward
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('strided,B,T', [(True, 4, 27), (True, 2, 108), (False, 2, 40)],
                         ids=['strided', 'strided_T108', 'dilated'])
def test_single_pass_is_bitwise_eval_backward(strided, B, T, core):
    m = _model(17, [3, 3, 3], 32, strided)
    x = torch.from_numpy(synth.synth_input(B, T, 17, 2, seed=2)).cuda()
    with torch.no_grad():
        T_out = m(x).shape[1]
    dy = torch.randn(B, T_out, 17, 3, generator=torch.Generator().manual_seed(3)).cuda()
    y0, g0 = _run(m, x, dy)
    for mf in (B * T_out, B * T_out + 7):
        y1, g1 = _run(m, x, dy, mf)
        assert torch.equal(y1, y0)
        _assert_same(g1, g0, exact=strided)


@pytest.mark.parametrize('strided,causal,B,T', [(True, False, 3, 81), (False, False, 2, 60), (False, True, 2, 60),
                                                (False, False, 5, 27)],
                         ids=['strided', 'dilated', 'causal', 'dilated_rf'])
def test_single_pass_workspace_is_eval_backward_workspace(strided, causal, B, T):
    m = _model(17, [3, 3, 3], 32, strided, causal)
    h = engine.model_handle(m, torch.device('cuda'))
    sn = engine._strided_now(m, T)
    T_out = h.lib.gast_out_frames(h.h, T, sn)
    need = h.lib.gast_eval_backward_workspace_bytes(h.h, B, T, sn)
    assert T_out > 0 and need > 0
    for mf in (B * T_out, B * T_out + 7):
        assert h.lib.gast_chunked_workspace_bytes(h.h, B, T, sn, mf, 1) == need, mf


# ---------------------------------------------------------------------------------------------------------------
# several passes: against the unchunked call, against fp64 at kink-free points, run to run
# ---------------------------------------------------------------------------------------------------------------
EXTRA_CASES = {
    'dilated_T45_j17_c32_eval': K.Case(17, [3, 3, 3], 32, 2, 45, False, False, False, False),
    'strided_T81_j17_c32_eval': K.Case(17, [3, 3, 3], 32, 3, 81, True, False, False, False),
}


@functools.lru_cache(maxsize=None)
def _reference(name):
    """K.reference for the cases of tests/kinkfree.py and those above"""
    if name in K.CASES:
        return K.CASES[name], K.reference(name)
    case = EXTRA_CASES[name]
    x = K.inputs(case)
    sd, marg = K.make_kink_free(K.module(case).state_dict(), x, case)
    with torch.no_grad():
        shape = K.port_forward({k: (v.double() if v.dtype.is_floating_point else v) for k, v in sd.items()},
                               x.double(), case).shape
    tgt = K.target(shape)
    y, loss, grads, scales = K.port_grads(sd, x, tgt, case, torch.float64)
    return case, dict(sd=sd, x=x, target=tgt, margins=marg, y=y, loss=loss, grads=grads, scales=scales)


MULTI = [  # kink-free case, max_frames
    ('causal_T40_j19_c16_eval', 5),      # 14 outputs per clip: windows of 5, 5, 4
    ('causal_T40_j19_c16_eval', 1),      # windows of one output frame
    ('dilated_T45_j17_c32_eval', 4),     # 19 outputs per clip: windows of 4 (x4) and 3
    ('strided_T81_j17_c32_eval', 2),     # strided, T > receptive field: windows of 2 and 1 output frames
    ('o1f_j17_c128_eval', 3),            # 8 clips of 1 output: passes of 3, 3, 2 whole clips
    ('fw5_dilated_j16_c32_eval', 2),     # dilated at T == receptive field (strided schedule): 2, 1 clips
]


def _loss_grads(m, ref, max_frames):
    m.zero_grad(set_to_none=True)
    x = ref['x'].cuda().requires_grad_()
    y = m(x) if max_frames is None else engine.run_model_chunked(m, x, max_frames)
    loss = _mpjpe(y, ref['target'].cuda())
    loss.backward()
    got = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    got['x'] = x.grad.detach().clone()
    return y.detach(), got


@pytest.mark.parametrize('name,max_frames', MULTI, ids=['%s_mf%d' % t for t in MULTI])
def test_multi_pass_gradients(name, max_frames, core):
    case, ref = _reference(name)
    relu, leaky, _ = ref['margins']
    assert relu >= K.MARGIN and leaky >= K.MARGIN, (relu, leaky)
    m = K.module(case)
    m.load_state_dict(ref['sd'])
    m = m.cuda().eval()
    y0, g0 = _loss_grads(m, ref, None)
    y1, g1 = _loss_grads(m, ref, max_frames)
    assert y1.shape[1] * case.B > max_frames, 'one pass: not a multi-pass case'
    assert torch.equal(y1, y0)
    # against the unchunked call: summation order only (bars of the FFMA core against fp64)
    err = K.errors({k: v.cpu().double() for k, v in g1.items()}, {k: v.cpu().double() for k, v in g0.items()},
                   ref['scales'])
    far = [(k, e) for k, e in err.items() if e[0] is not None and (e[0] > K.L2_BAR['ffma'] or e[1] > K.MAX_BAR['ffma'])]
    assert not far, far
    # against fp64 at the kink-free point: the rounding-level bars of the unchunked gradients
    bad, _ = K.check({k: v.cpu().double() for k, v in g1.items()}, ref['grads'], ref['scales'],
                     'ffma' if core == 1 else 'tc')
    assert not bad, sorted(bad, key=lambda t: -(t[1] or 0))[:12]
    # run to run (bit for bit on the strided schedule)
    y2, g2 = _loss_grads(m, ref, max_frames)
    assert torch.equal(y2, y1)
    _assert_same(g2, g1, exact=case.strided or case.T == m.receptive_field())


# ---------------------------------------------------------------------------------------------------------------
# TF32 training precision, input-only gradients, accumulation into .grad
# ---------------------------------------------------------------------------------------------------------------
def test_tf32_training_precision():
    m = _model(17, [3, 3, 3], 64, strided=True)
    engine.set_training_precision(m, 'tf32')
    x = torch.from_numpy(synth.synth_input(2, 108, 17, 2, seed=4)).cuda()
    dy = torch.randn(2, 4, 17, 3, generator=torch.Generator().manual_seed(5)).cuda()
    y0, g0 = _run(m, x, dy)
    assert _handle(m).wgrad_tc_launches() > 0
    y1, g1 = _run(m, x, dy, 8)                      # one pass
    assert torch.equal(y1, y0)
    _assert_bitwise(g1, g0)
    _, g2 = _run(m, x, dy, 3)                       # windows of 3 and 1 output frames
    assert _handle(m).wgrad_tc_launches() > 0
    _, g3 = _run(m, x, dy, 3)
    _assert_bitwise(g3, g2)
    # summation order only; a gradient that is a cancelling sum is held to the largest gradient entry instead
    top = max(v.abs().max().item() for v in g0.values())
    for k in g0:
        rel = ((g2[k] - g0[k]).norm() / g0[k].norm().clamp_min(1e-30)).item()
        assert rel < 1e-3 or (g2[k] - g0[k]).abs().max().item() <= 1e-5 * top, (k, rel)


def test_input_only_gradient_runs_no_weight_gradients(core):
    x = torch.from_numpy(synth.synth_input(2, 40, 17, 2, seed=6)).cuda()
    dy = torch.randn(2, 14, 17, 3, generator=torch.Generator().manual_seed(7)).cuda()
    m = _model(17, [3, 3, 3], 32)
    _, g_full = _run(m, x, dy, 5)
    n_full = _handle(m).launches()
    m.requires_grad_(False)
    _, g_x = _run(m, x, dy, 5)
    n_x = _handle(m).launches()
    assert list(g_x) == ['x'] and all(p.grad is None for p in m.parameters())
    assert (g_x['x'] - g_full['x']).abs().max().item() <= 1e-6 * g_full['x'].abs().max().item()
    assert n_x < n_full, (n_x, n_full)


def test_accumulates_into_existing_grad(core):
    m = _model(17, [3, 3, 3], 32, strided=True)      # the strided schedule: the gradients repeat bit for bit
    x = torch.from_numpy(synth.synth_input(2, 81, 17, 2, seed=8)).cuda()
    dy = torch.randn(2, 3, 17, 3, generator=torch.Generator().manual_seed(9)).cuda()
    _, g = _run(m, x, dy, 2)
    for i, p in enumerate(m.parameters()):
        p.grad = torch.full_like(p, 0.25 + i)
    engine.run_model_chunked(m, x, 2).backward(dy)
    for i, (k, p) in enumerate(m.named_parameters()):
        assert torch.equal(p.grad, torch.full_like(p, 0.25 + i) + g[k]), k


# ---------------------------------------------------------------------------------------------------------------
# errors and refusals
# ---------------------------------------------------------------------------------------------------------------
def test_version_check_and_train_mode():
    m = _model(17, [3, 3, 3], 32)
    x = torch.from_numpy(synth.synth_input(2, 40, 17, 2, seed=1)).cuda().requires_grad_()
    y = engine.run_model_chunked(m, x, 5)
    with torch.no_grad():
        x.add_(1.0)
    with pytest.raises(RuntimeError, match='inplace'):
        y.sum().backward()
    y = engine.run_model_chunked(m, x.detach(), 5)
    with torch.no_grad():
        m.layers_bn[0].running_var.mul_(1.0)
    with pytest.raises(RuntimeError, match='inplace'):
        y.sum().backward()
    m.train()
    with pytest.raises(engine.GastError, match='train mode'):
        engine.run_model_chunked(m, x.detach(), 5)
    with pytest.raises(engine.GastError, match='train mode'):
        with torch.no_grad():
            engine.run_model_chunked(m, x.detach(), 5)


def test_refused_calls_change_no_buffer():
    m = _model(17, [3, 3, 3], 32)
    B, T, T_out = 2, 40, 14
    x = torch.from_numpy(synth.synth_input(B, T, 17, 2, seed=1)).cuda()
    with torch.no_grad():
        m(x)
    h = _handle(m)
    lib = h.lib
    names = [k for k, _ in engine.named_params(m)]
    bufs = {k: torch.full_like(p, 7.0) for k, p in engine.named_params(m)}
    engine._bind(h, 'gast_bind_grads', list(bufs.items()))
    dy = torch.ones(B, T_out, 17, 3, device='cuda')
    dx = torch.full_like(x, 7.0)
    y = torch.full((B, T_out, 17, 3), 7.0, device='cuda')
    need = int(lib.gast_chunked_workspace_bytes(h.h, B, T, 0, 5, 1))
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')

    def back(mf, nbytes, param_grads=1):
        return lib.gast_eval_backward_chunked(h.h, _p(x), _p(dy), _p(dx), param_grads, B, T, 0, mf, _p(ws), nbytes,
                                              _st())

    def untouched():
        torch.cuda.synchronize()
        return (torch.all(dx == 7.0).item() and torch.all(y == 7.0).item() and
                all(torch.all(b == 7.0).item() for b in bufs.values()))

    assert back(5, need - 1) != 0 and 'workspace too small' in engine.L.last_error()
    assert back(0, need) != 0 and 'max_frames' in engine.L.last_error()
    assert lib.gast_chunked_workspace_bytes(h.h, B, T, 0, 0, 1) == 0
    assert lib.gast_eval_backward_chunked(h.h, _p(x), _p(dy), _p(dx), 1, 0, T, 0, 5, _p(ws), need, _st()) != 0
    assert lib.gast_eval_backward_chunked(h.h, _p(x), _p(dy), _p(dx), 1, B, 10, 0, 5, _p(ws), need, _st()) != 0
    fwd_need = int(lib.gast_chunked_workspace_bytes(h.h, B, T, 0, 5, 0))
    assert lib.gast_forward_chunked(h.h, _p(x), _p(y), B, T, 0, 5, _p(ws), fwd_need - 1, _st()) != 0
    assert lib.gast_forward_chunked(h.h, _p(x), _p(y), B, T, 0, 0, _p(ws), fwd_need, _st()) != 0
    assert untouched()
    # a gradient buffer of the wrong size is refused, naming its key; the input-only call does not need it
    key = names[3]
    engine._bind(h, 'gast_bind_grads', [(key, torch.zeros(bufs[key].numel() + 1, device='cuda'))])
    assert back(5, need) != 0 and key in engine.L.last_error()
    assert untouched()
    assert back(5, need, param_grads=0) == 0
    torch.cuda.synchronize()
    assert not torch.all(dx == 7.0).item() and all(torch.all(b == 7.0).item() for b in bufs.values())


def test_workspace_query_stops_growing_with_T_or_B():
    m = _model(17, [3, 3, 3], 32)
    with torch.no_grad():
        m(torch.from_numpy(synth.synth_input(1, 27, 17, 2, seed=1)).cuda())
    h = _handle(m)
    q = h.lib.gast_chunked_workspace_bytes
    for wb in (0, 1):
        # windows: one clip needs several passes at any of these T
        sizes = {q(h.h, 1, T, 0, 8, wb) for T in (40, 100, 1000, 100000)} | {q(h.h, 5, 1000, 0, 8, wb)}
        assert len(sizes) == 1 and 0 not in sizes, sizes
        # whole clips (T == receptive field, strided schedule, one output each): 8 per pass.  A one-pass backward
        # takes no pass-gradient area, so its query stops growing at two passes
        full = {q(h.h, B, 27, 1, 8, wb) for B in ((8,) if wb == 0 else ()) + (9, 16, 100, 10000)}
        assert len(full) == 1 and 0 not in full, full
        assert q(h.h, 4, 27, 1, 8, wb) <= q(h.h, 8, 27, 1, 8, wb) <= min(full)
    assert q(h.h, 1, 1000, 0, 8, 0) < q(h.h, 1, 1000, 0, 8, 1)


# ---------------------------------------------------------------------------------------------------------------
# a recording too long for the unchunked backward
# ---------------------------------------------------------------------------------------------------------------
def test_recording_beyond_device_memory_completes_chunked():
    m = _model(17, [3, 3, 3], 128)
    rf = m.receptive_field()
    with torch.no_grad():
        m(torch.from_numpy(synth.synth_input(1, rf, 17, 2, seed=1)).cuda())
    h = _handle(m)
    total = torch.cuda.get_device_properties(0).total_memory
    q = lambda T: int(h.lib.gast_eval_backward_workspace_bytes(h.h, 1, T, 0))
    per_frame = (q(rf + 2000) - q(rf + 1000)) / 1000.0
    T = int(1.05 * total / per_frame) + rf
    assert q(T) > total, (q(T), total)             # the unchunked call could not even get its workspace
    mf = 2048
    params = sum(p.numel() for p in m.parameters()) * 4
    ws_chunked = int(h.lib.gast_chunked_workspace_bytes(h.h, 1, T, 0, mf, 1))
    # one window's unchunked workspace, and the pass-gradient area
    assert 0 < ws_chunked < q(mf + rf) + params + (64 << 20)
    x = torch.from_numpy(synth.synth_input(1, T, 17, 2, seed=2)).cuda().requires_grad_()
    dy = torch.randn(1, T - rf + 1, 17, 3, generator=torch.Generator().manual_seed(3)).cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    y = engine.run_model_chunked(m, x, mf)
    y.backward(dy)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    # the backward's workspace, dx, the flat gradient buffer and the .grad tensors, y, and allocator rounding
    bound = ws_chunked + x.numel() * 4 + 2 * params + 2 * y.numel() * 4 + (64 << 20)
    assert peak < bound, (peak, bound, ws_chunked)
    assert torch.isfinite(x.grad).all() and x.grad.abs().max().item() > 0
    assert all(torch.isfinite(p.grad).all() for p in m.parameters())
    # the first window's outputs are those of the unchunked call on that window alone
    with torch.no_grad():
        y_head = m(x.detach()[:, :mf + rf - 1])
    assert torch.equal(y.detach()[:, :mf], y_head)
