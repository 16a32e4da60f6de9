"""GPU: a training or gradient call refuses a bad parameter or gradient-buffer binding before its first launch.

The refused training forward leaves the running statistics and its output untouched; the refused backward keeps the
saved forward, so the caller can fix the binding and differentiate that forward.  The workspace queries do not need
anything bound."""
import ctypes as C

import pytest
import torch

from gast_b200 import engine, synth

pytestmark = pytest.mark.gpu

B, T, J = 4, 27, 17


def _model():
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModelOptimized1f
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    m = SpatioTemporalModelOptimized1f(adj, J, 2, J, [3, 3, 3], dropout=0.0, channels=32)
    synth.randomize_module(m, 5)
    return m.cuda().train()


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else None)


def _st():
    return C.c_void_p(engine._stream(torch.device('cuda')))


def _setup():
    m = _model()
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=3)).cuda()
    h = engine.model_handle(m, x.device)
    h.bind_only(m)
    need = int(h.lib.gast_train_workspace_bytes(h.h, B, T, C.c_float(0.0)))
    assert need > 0
    ws = torch.empty(need, dtype=torch.uint8, device='cuda')
    y = torch.empty((B, 1, J, 3), device='cuda')
    return m, x, h, ws, y, need


def _forward(h, x, y, ws, need):
    return h.lib.gast_forward_train(h.h, _p(x), _p(y), B, T, C.c_float(0.0), C.c_uint64(0), _p(ws), need, _st())


def _backward(h, dy, dx, param_grads, ws, need):
    return h.lib.gast_backward_input(h.h, _p(dy), _p(dx), param_grads, _p(ws), need, _st())


def _bind_one(h, entry, key, numel):
    engine._bind(h, entry, [(key, torch.zeros(numel, device='cuda'))])


def _nan_grads(m):
    """one NaN-filled gradient buffer per parameter, by key"""
    return {k: torch.full_like(p, float('nan')) for k, p in engine.named_params(m)}


def _bind_grads(h, grads):
    engine._bind(h, 'gast_bind_grads', list(grads.items()))


def _running(m):
    return {k: v.clone() for k, v in m.state_dict().items() if 'running_' in k}


def test_forward_train_refuses_bad_parameter_before_any_launch():
    m, x, h, ws, y, need = _setup()
    assert _forward(h, x, y, ws, need) == 0
    n = h.launches()
    torch.cuda.synchronize()
    y0, run0 = y.clone(), _running(m)
    _bind_one(h, 'gast_bind', 'shrink.weight', m.shrink.weight.numel() + 1)   # the last key the forward reads
    assert _forward(h, x, y, ws, need) != 0 and 'shrink.weight' in engine.L.last_error()
    torch.cuda.synchronize()
    assert h.launches() == n
    assert torch.equal(y, y0)
    run1 = _running(m)
    assert all(torch.equal(run0[k], run1[k]) for k in run0), 'a refused forward updated the running statistics'
    h.bind_only(m)
    assert _forward(h, x, y, ws, need) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(y).all()


def test_backward_refuses_bad_gradient_buffer_and_keeps_the_saved_forward():
    m, x, h, ws, y, need = _setup()
    dy = torch.from_numpy(synth.synth_target(B, J, seed=4)).cuda()
    # an uninterrupted step
    ref = _nan_grads(m)
    dx_ref = torch.empty_like(x)
    _bind_grads(h, ref)
    assert _forward(h, x, y, ws, need) == 0
    assert _backward(h, dy, dx_ref, 1, ws, need) == 0
    # the same step, first with init_bn.bias (the last gradient the backward writes) bound at the wrong size
    grads = _nan_grads(m)
    dx = torch.full_like(x, float('nan'))
    _bind_grads(h, grads)
    _bind_one(h, 'gast_bind_grads', 'init_bn.bias', m.init_bn.bias.numel() + 1)
    assert _forward(h, x, y, ws, need) == 0
    n = h.launches()
    assert _backward(h, dy, dx, 1, ws, need) != 0 and 'init_bn.bias' in engine.L.last_error()
    torch.cuda.synchronize()
    assert h.launches() == n
    assert all(torch.isnan(g).all() for g in grads.values()) and torch.isnan(dx).all()
    _bind_grads(h, {'init_bn.bias': grads['init_bn.bias']})
    assert _backward(h, dy, dx, 1, ws, need) == 0
    torch.cuda.synchronize()
    assert torch.equal(dx, dx_ref)
    assert all(torch.equal(grads[k], ref[k]) for k in ref)
    # without parameter gradients the gradient buffers are not read, so a bad one does not matter
    _bind_one(h, 'gast_bind_grads', 'init_bn.bias', m.init_bn.bias.numel() + 1)
    assert _forward(h, x, y, ws, need) == 0
    dx.fill_(float('nan'))
    assert _backward(h, dy, dx, 0, ws, need) == 0
    torch.cuda.synchronize()
    assert torch.equal(dx, dx_ref)


def test_eval_backward_refuses_bad_bindings_before_any_launch():
    m, x, h, ws, y, need = _setup()
    m.eval()
    dy = torch.from_numpy(synth.synth_target(B, J, seed=4)).cuda()
    need = int(h.lib.gast_eval_backward_workspace_bytes(h.h, B, T, 1))
    ews = torch.empty(need, dtype=torch.uint8, device='cuda')
    grads = _nan_grads(m)
    _bind_grads(h, grads)
    dx = torch.full_like(x, float('nan'))

    def call():
        return h.lib.gast_eval_backward(h.h, _p(x), _p(dy), _p(dx), 1, B, T, 1, _p(ews), need, _st())

    assert _forward(h, x, y, ws, ws.numel()) == 0
    n = h.launches()
    _bind_one(h, 'gast_bind', 'shrink.weight', m.shrink.weight.numel() - 1)
    assert call() != 0 and 'shrink.weight' in engine.L.last_error()
    assert h.launches() == n
    h.bind_only(m)
    _bind_one(h, 'gast_bind_grads', 'init_bn.bias', m.init_bn.bias.numel() + 1)
    assert call() != 0 and 'init_bn.bias' in engine.L.last_error()
    assert h.launches() == n
    torch.cuda.synchronize()
    assert all(torch.isnan(g).all() for g in grads.values()) and torch.isnan(dx).all()
    _bind_grads(h, {'init_bn.bias': grads['init_bn.bias']})
    assert call() == 0
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all() and all(torch.isfinite(g).all() for g in grads.values())


def test_workspace_queries_need_no_binding():
    m = _model()
    h = engine.model_handle(m, m.shrink.weight.device)

    def sizes():
        return ([int(h.lib.gast_train_workspace_bytes(h.h, b, t, C.c_float(p)))
                 for b, t, p in ((1, 27, 0.0), (4, 27, 0.25), (64, 81, 0.05))] +
                [int(h.lib.gast_eval_backward_workspace_bytes(h.h, b, t, 1)) for b, t in ((1, 27), (16, 81))])

    unbound = sizes()
    assert all(s > 0 for s in unbound)
    h.bind_only(m)
    _bind_grads(h, _nan_grads(m))
    assert sizes() == unbound
