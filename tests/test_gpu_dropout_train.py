"""Training with dropout on the GPU against the fp64 port with the library's own masks (tests/dropoutref.py restates
dropout_mask_kernel): the train-mode output and the running statistics downstream of the masks, two outstanding
dropout forwards each differentiated with its own masks, a CUDA-graph replay's masks (the device-side counter),
three SGD steps, and the refusal of p = 1.  The per-tensor gradient checks of the dropout cases are
tests/test_gpu_grad_exact.py's (kinkfree.CASES); both GEMM cores."""
import pytest
import torch

from gast_b200 import engine, synth
import dropoutref as D
import kinkfree as K
from test_gpu_train import _adj, check_three_sgd_steps

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def _mpjpe(y, t):
    return torch.mean(torch.norm(y - t, dim=3))


@pytest.mark.parametrize('name', ['o1f_j17_c128_train_drop05', 'causal_T40_j17_c48_train_drop25'])
def test_forward_and_running_statistics(name, core):
    """y at the kink-free point and every running statistic after the step, against the fp64 port with the masks;
    the same step without dropout gives another y"""
    case = K.CASES[name]
    ref = K.reference(name)
    sd64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in ref['sd'].items()}
    stats = {}
    with torch.no_grad():
        y_ref = K.port_forward(sd64, ref['x'].double(), case, stats=stats)
    assert len(stats) == 2 * sum(1 for k in sd64 if k.endswith('running_mean'))
    m = K.module(case)
    m.load_state_dict(ref['sd'])
    m = m.cuda().train()
    x = ref['x'].cuda()
    torch.manual_seed(K.DROP_SEED)
    with torch.no_grad():
        y = m(x).cpu().double()
    assert (y - y_ref).abs().max().item() <= K.Y_BAR * y_ref.abs().max().item()
    sd = m.state_dict()
    for k, v in stats.items():
        err = (sd[k].cpu().double() - v).abs().max().item()
        assert err <= 1e-5 * max(1.0, v.abs().max().item()), (k, err)
    m0 = K.module(case._replace(drop=0.0))
    m0.load_state_dict(ref['sd'])
    with torch.no_grad():
        y0 = m0.cuda().train()(x).cpu().double()
    assert (y0 - y).abs().max().item() > 1e-2 * y.abs().max().item()


def test_two_outstanding_dropout_forwards(core):
    """two dropout forwards with different seeds, one backward of their sum: the sum of each differentiated alone,
    so each backward reads the masks of its own workspace"""
    from model.gast_net import SpatioTemporalModelOptimized1f
    m = SpatioTemporalModelOptimized1f(_adj(17), 17, 2, 17, [3, 3, 3], dropout=0.25, channels=32)
    synth.randomize_module(m, 3)
    m = m.cuda().train()
    xa = torch.from_numpy(synth.synth_input(4, 27, 17, 2, seed=1)).cuda()
    xb = torch.from_numpy(synth.synth_input(4, 27, 17, 2, seed=2)).cuda()

    def grads(x, seed):
        m.zero_grad()
        torch.manual_seed(seed)
        m(x).square().sum().backward()
        return [p.grad.clone() for p in m.parameters()]
    ga, gb = grads(xa, 11), grads(xb, 12)
    assert any(not torch.allclose(a, b, rtol=1e-2) for a, b in zip(grads(xa, 12), ga))   # the masks matter
    m.zero_grad()
    torch.manual_seed(11)
    ya = m(xa)
    torch.manual_seed(12)
    yb = m(xb)
    (ya.square().sum() + yb.square().sum()).backward()
    for p, a, b in zip(m.parameters(), ga, gb):
        assert torch.allclose(p.grad, a + b, rtol=1e-4, atol=1e-6 * float((a + b).abs().max() + 1e-30))


def test_graph_replay_uses_the_counted_masks(core, monkeypatch):
    """GraphedTrainer at p = 0.05: a replay applies the masks of the captured seed plus the device counter as read
    before the replay (three warm-up forwards, one bump each), every gradient at rounding-level bars against the fp64
    port at a kink-free point for those masks, and the counter advances by one step"""
    from gast_b200.trainer import GraphedTrainer
    name = 'o1f_j17_c128_train_drop05'
    case = K.CASES[name]
    seeds = []
    real = torch.randint

    def randint(*a, **kw):
        r = real(*a, **kw)
        if a[:2] == (0, 2 ** 62):
            seeds.append(int(r.item()))
        return r
    monkeypatch.setattr(torch, 'randint', randint)
    x = K.inputs(case)
    tgt = K.target((case.B, 1, case.J, 3))
    m = K.module(case).cuda()
    tr = GraphedTrainer(m, lambda ps: torch.optim.SGD(ps, lr=0.0), tuple(x.shape), tuple(tgt.shape))
    assert len(seeds) == 4                                   # three warm-up forwards and the captured one
    dstate = D.dstate_value(m.__dict__['_gast_dropout_state'])
    assert dstate == (3 * D.DSTATE_STEP) & D.U64
    masks = D.masks(case, case.B, case.T, case.J, case.drop, seeds[-1], dstate)
    sd, (relu, leaky, _) = K.make_kink_free({k: v.detach().cpu() for k, v in m.state_dict().items()}, x, case, masks)
    assert relu >= K.MARGIN and leaky >= K.MARGIN, (relu, leaky)
    with torch.no_grad():
        for k, p in m.named_parameters():
            p.copy_(sd[k])                                   # in place: the graph keeps the pointers
    tr.x.copy_(x)
    tr.y.copy_(tgt)
    tr.graph.replay()
    _, loss, grads, scales = K.port_grads(sd, x, tgt, case, torch.float64, masks)
    grads.pop('x')
    got = {k: p.grad.cpu().double() for k, p in m.named_parameters()}
    bad, _ = K.check(got, grads, scales, 'ffma' if core == 1 else 'tc')
    assert not bad, sorted(bad, key=lambda t: -(t[1] or 0))[:12]
    assert abs(float(tr.loss) - loss) <= K.LOSS_BAR * abs(loss)
    assert D.dstate_value(m.__dict__['_gast_dropout_state']) == (4 * D.DSTATE_STEP) & D.U64
    assert len(seeds) == 4                                   # a replay draws no new seed


def test_three_sgd_steps_with_dropout(core):
    """test_gpu_train.test_three_sgd_steps_match_reference_port at the reference's default p = 0.05, the port
    replaying each step's masks"""
    check_three_sgd_steps(0.05)


def test_dropout_one_is_refused():
    """p = 1 has no scale: a train-mode forward raises instead of returning zeros"""
    from model.gast_net import SpatioTemporalModelOptimized1f
    m = SpatioTemporalModelOptimized1f(_adj(17), 17, 2, 17, [3, 3, 3], dropout=1.0, channels=32)
    synth.randomize_module(m, 3)
    m = m.cuda().train()
    with pytest.raises(engine.GastError, match='dropout'):
        m(torch.from_numpy(synth.synth_input(2, 27, 17, 2)).cuda())
