"""GPU: the checks every model call makes before its first launch, and the launch counters it restarts.

A training forward refuses an empty batch; a backward refuses a workspace smaller than its forward checked, before it
writes anything and without losing the saved forward; after a training step the tensor-core count covers that step
alone."""
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


def _train_forward(h, x, y, ws, ws_bytes, batch=B):
    return h.lib.gast_forward_train(h.h, _p(x), _p(y), batch, T, C.c_float(0.0), C.c_uint64(0), _p(ws), ws_bytes,
                                    C.c_void_p(engine._stream(ws.device)))


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


def test_forward_train_refuses_empty_batch_and_null_pointers():
    m, x, h, ws, y, need = _setup()
    assert _train_forward(h, x, y, ws, need) == 0
    n = h.launches()
    assert _train_forward(h, x, y, ws, need, batch=0) != 0 and 'empty batch' in engine.L.last_error()
    assert _train_forward(h, None, y, ws, need) != 0 and 'device pointers' in engine.L.last_error()
    assert _train_forward(h, x, None, ws, need) != 0 and 'device pointers' in engine.L.last_error()
    assert h.launches() == n                      # refused before any launch: the counts are the last call's
    torch.cuda.synchronize()


def test_backward_refuses_short_workspace_before_any_launch():
    m, x, h, ws, y, need = _setup()
    assert _train_forward(h, x, y, ws, need) == 0
    n_fwd = h.launches()
    dy = torch.ones_like(y)
    dx = torch.empty_like(x)
    st = C.c_void_p(engine._stream(x.device))
    rc = h.lib.gast_backward_input(h.h, _p(dy), _p(dx), 0, _p(ws), need - 1, st)
    assert rc != 0 and 'workspace too small' in engine.L.last_error()
    assert h.launches() == n_fwd
    rc = h.lib.gast_backward_input(h.h, None, _p(dx), 0, _p(ws), need, st)
    assert rc != 0 and 'dy' in engine.L.last_error()
    assert h.launches() == n_fwd
    # the refusals left the saved forward in place: the backward at full size runs and continues the forward's count
    assert h.lib.gast_backward_input(h.h, _p(dy), _p(dx), 0, _p(ws), need, st) == 0
    assert h.launches() > n_fwd
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all()


def test_tc_count_covers_one_training_step():
    m = _model()
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=3)).cuda()
    h = engine.model_handle(m, x.device)
    counts = []
    for _ in range(2):
        m(x).sum().backward()
        counts.append((h.launches(), int(h.lib.gast_last_tc_launch_count(h.h))))
        with torch.no_grad():
            m.eval()(x)                          # an eval forward in between restarts every count
            assert 0 < int(h.lib.gast_last_tc_launch_count(h.h)) <= h.launches()
            m.train()
    torch.cuda.synchronize()
    assert counts[0] == counts[1] and counts[0][1] > 0, counts
