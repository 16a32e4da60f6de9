"""Training steps and gradients repeat bit for bit on every schedule: the strided one (Optimized1f), the dilated one
(causal or not) and the dense ablation, on both GEMM cores and in both training precisions.  The backward adds the
overlapping taps of a temporal conv by a gather from the input side (seg_adjoint_kernel) and takes every column sum
(BatchNorm statistics, their gradients, the bias gradients) in a fixed order, so nothing depends on how the hardware
schedules blocks:
  * a train-mode step with dropout, from one state_dict, on one batch, under one torch.manual_seed: y, the loss,
    every parameter gradient, every running statistic and num_batches_tracked;
  * eval-mode gradients (dL/dx and every parameter gradient) of a ~2,000-frame recording through model(x) and
    engine.run_model_chunked (windows that do not divide T_out, and passes of whole clips); a chunked call of one pass
    is bitwise the unchunked call;
  * GraphedTrainer against DataParallelTrainer on a dilated model: three FusedAdam steps give the same parameters.
The largest cases (128 channels, b = 64 at T = rf + 26, and the recording) have 256 row blocks per column sum and
up to three taps per input frame."""
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


@pytest.fixture(params=['fp32', 'tf32'])
def tprec(request):
    return request.param


def _mpjpe(y, t):
    return torch.mean(torch.norm(y - t, dim=3))


def _assert_bitwise(a, b):
    assert a.keys() == b.keys()
    for k in a:
        assert torch.equal(a[k], b[k]), k


# J, fw, ch, B, T, strided, causal, dense (train mode, dropout 0.25)
TRAIN = {
    'o1f_c128_b64': K.Case(17, [3, 3, 3], 128, 64, 27, True, False, False, True, 0.25),
    'dilated_c128_b64_T53': K.Case(17, [3, 3, 3], 128, 64, 53, False, False, False, True, 0.25),
    'causal_3333_c64_b8_T100': K.Case(17, [3, 3, 3, 3], 64, 8, 100, False, True, False, True, 0.25),
    'dense_c32_b16_T40': K.Case(17, [3, 3, 3], 32, 16, 40, False, False, True, True, 0.25),
}


@pytest.mark.parametrize('name', list(TRAIN))
def test_train_step_repeats(name, core, tprec):
    case = TRAIN[name]
    m = engine.set_training_precision(K.module(case).cuda(), tprec)
    x = torch.from_numpy(synth.synth_input(case.B, case.T, case.J, 2, seed=1)).cuda()
    sd = {k: v.clone() for k, v in m.state_dict().items()}

    def step():
        m.load_state_dict(sd)
        m.train()
        m.zero_grad(set_to_none=True)
        torch.manual_seed(7)
        y = m(x)
        tgt = torch.randn(y.shape, generator=torch.Generator().manual_seed(3)).cuda()
        loss = _mpjpe(y, tgt)
        loss.backward()
        out = {'y': y.detach().clone(), 'loss': loss.detach().clone()}
        out.update({'grad.' + k: p.grad.detach().clone() for k, p in m.named_parameters()})
        out.update({'state.' + k: v.detach().clone() for k, v in m.state_dict().items()})
        return out
    a, b = step(), step()
    _assert_bitwise(a, b)
    # the step did train: every running statistic moved, and the masks took effect
    assert all(not torch.equal(a['state.' + k], sd[k]) for k in sd if k.endswith('running_mean'))
    m.load_state_dict(sd)
    m.train()
    torch.manual_seed(8)
    with torch.no_grad():
        assert not torch.equal(m(x), a['y'])


# ---------------------------------------------------------------------------------------------------------------
# eval mode: model(x) and run_model_chunked
# ---------------------------------------------------------------------------------------------------------------
EVAL = {  # J, fw, ch, strided, causal, dense; recording frames; (clips, frames) of the whole-clip call
    'o1f_c128': (K.Case(17, [3, 3, 3], 128, 1, 1, True, False, False, False), 2000, (6, 27 * 2 + 5)),
    'dilated_c128': (K.Case(17, [3, 3, 3], 128, 1, 1, False, False, False, False), 2000, (6, 37)),
    'causal_3333_c64': (K.Case(17, [3, 3, 3, 3], 64, 1, 1, False, True, False, False), 2000, (5, 90)),
    'dense_c32': (K.Case(17, [3, 3, 3], 32, 1, 1, False, False, True, False), 2000, (6, 40)),
}


def _run(m, x, dy, max_frames=None):
    """y and every gradient of (y * dy).sum(), dL/dx included, through model(x) or run_model_chunked"""
    m.zero_grad(set_to_none=True)
    xx = x.clone().requires_grad_()
    y = m(xx) if max_frames is None else engine.run_model_chunked(m, xx, max_frames)
    y.backward(dy)
    g = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    g['x'] = xx.grad.detach().clone()
    g['y'] = y.detach().clone()
    return g


@pytest.mark.parametrize('name', list(EVAL))
def test_eval_gradients_repeat(name, core, tprec):
    case, T, (Bc, Tc) = EVAL[name]
    m = engine.set_training_precision(K.module(case).cuda().eval(), tprec)
    for B, TT, seed in ((1, T, 1), (Bc, Tc, 2)):
        x = torch.from_numpy(synth.synth_input(B, TT, case.J, 2, seed=seed)).cuda()
        with torch.no_grad():
            T_out = m(x).shape[1]
        dy = torch.randn(B, T_out, case.J, 3, generator=torch.Generator().manual_seed(seed)).cuda()
        whole = _run(m, x, dy)
        _assert_bitwise(_run(m, x, dy), whole)
        # one pass is the unchunked call
        _assert_bitwise(_run(m, x, dy, B * T_out), whole)
        if B == 1:
            mf = T_out // 4 + 3                   # windows that do not divide T_out
            assert T_out % mf != 0
        else:
            mf = 2 * T_out                        # passes of two whole clips
            assert B * T_out > mf
        chunked = _run(m, x, dy, mf)
        _assert_bitwise(_run(m, x, dy, mf), chunked)
        assert torch.equal(chunked['y'], whole['y'])


# ---------------------------------------------------------------------------------------------------------------
# CUDA-graph replay against the eager trainer
# ---------------------------------------------------------------------------------------------------------------
def test_graphed_trainer_matches_eager(core, tprec):
    """dropout 0: the graphed trainer draws its masks from the device counter, the eager one from torch's seed"""
    from gast_b200.trainer import DataParallelTrainer, GraphedTrainer
    from gast_b200.pipeline import FusedAdam
    case = K.Case(17, [3, 3, 3], 64, 32, 40, False, False, False, True, 0.0)
    make = lambda: engine.set_training_precision(K.module(case).cuda(), tprec)  # noqa: E731
    opt = lambda ps: FusedAdam(ps, lr=1e-3, amsgrad=True)  # noqa: E731
    T_out = case.T - 27 + 1
    xs = [torch.from_numpy(synth.synth_input(case.B, case.T, case.J, 2, seed=40 + i)).cuda() for i in range(3)]
    ys = [torch.randn(case.B, T_out, case.J, 3, generator=torch.Generator().manual_seed(50 + i)).cuda()
          for i in range(3)]
    a = DataParallelTrainer(make(), opt)
    g = GraphedTrainer(make(), opt, tuple(xs[0].shape), tuple(ys[0].shape))
    g.model.load_state_dict(a.model.state_dict())       # in place: the graph keeps its pointers
    sd0 = {k: v.clone() for k, v in a.model.state_dict().items()}
    for x, y in zip(xs, ys):
        la, lg = a.step(x, y), g.step(x, y)
        assert torch.equal(la, lg)
    pa, pg = dict(a.model.named_parameters()), dict(g.model.named_parameters())
    for k in pa:
        assert torch.equal(pa[k], pg[k]), k
    assert any(not torch.equal(pa[k], sd0[k]) for k in pa)
