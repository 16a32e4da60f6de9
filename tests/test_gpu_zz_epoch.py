"""Whole training epochs on the device (gast_b200.training.EpochTrainer) against trainval.py's own loop:
  * the indexed gather serves every batch of an epoch, the tail included, as chunk_gather does for the host slice;
  * the indexed Adam step is gast_adam_step at the same step and lr, bit for bit;
  * two epochs with an lr decay between them equal the reference's unchanged main.train (oracle/_ref/) over the device
    ChunkedGenerator and FusedAdam, and over the reference's host ChunkedGenerator, bit for bit, for Optimized1f and
    the dilated model at chunk length > 1 on both GEMM cores and in both training precisions;
  * dropout masks repeat from the same counter and change from step to step; an epoch makes no host round trip;
    construction leaves no trace; eval_epoch is main.eval; a resumed run is the uninterrupted one; refusals."""
import copy
import io

import numpy as np
import pytest
import torch

from gast_b200 import engine, synth, training
from gast_b200 import pipeline as P
from gast_b200.engine import GastError
from test_unchanged_callers import LEFT, RIGHT, callers, needs_callers  # noqa: F401  (module fixture)
import epochref

pytestmark = pytest.mark.gpu

BETAS = (0.9, 0.999)
DECAY = 0.95


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def _split(n, lengths, seed, J=17):
    rs = np.random.RandomState(seed)
    p2 = [(0.5 * rs.standard_normal((T, J, 2))).astype(np.float32) for T in lengths[:n]]
    p3 = [(0.3 * rs.standard_normal((T, J, 3))).astype(np.float32) for T in lengths[:n]]
    return p2, p3


# name: model class, channels, chunk length, batch size (every case has a shorter last batch)
MODELS = {'o1f_27f': ('o1f', 32, 1, 40), 'dilated_27f_chunk4': ('dilated', 32, 4, 12)}
LENGTHS = [30, 41, 25]


def _model(kind, ch, drop=0.0, seed=4):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), LEFT, RIGHT))
    cls = SpatioTemporalModelOptimized1f if kind == 'o1f' else SpatioTemporalModel
    m = cls(adj, 17, 2, 17, [3, 3, 3], dropout=drop, channels=ch)
    synth.randomize_module(m, seed)
    return m.cuda().train()


def _dgen(p2, p3, chunk, B, seed=1234, **kw):
    from device.common.generators import ChunkedGenerator
    return ChunkedGenerator(B, None, p3, p2, chunk, pad=13, causal_shift=0, shuffle=True, random_seed=seed,
                            augment=True, kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT, **kw)


def _adam(m, lr=1e-3, **kw):
    return P.FusedAdam(m.parameters(), lr=lr, amsgrad=True, **kw)


def _state(m, opt):
    out = {'p.' + k: v.detach().clone() for k, v in m.state_dict().items()}
    out.update({'m1': opt.exp_avg.clone(), 'm2': opt.exp_avg_sq.clone()})
    if opt.max_exp_avg_sq is not None:
        out['m3'] = opt.max_exp_avg_sq.clone()
    out['step'] = opt.step_count
    return out


def _assert_same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def _decay(opt):
    for g in opt.param_groups:                                   # trainval.py:162-164
        g['lr'] *= DECAY


# ---------------------------------------------------------------------------------------------------------------
def test_indexed_gather_serves_every_batch():
    """flip augmentation, causal shift, chunk length > 1, 3D targets and cameras; a tail batch of 7"""
    from device.common.generators import ChunkedGenerator
    p2, p3 = _split(3, [30, 41, 25], 11)
    cams = [np.arange(9, dtype=np.float32) + i for i in range(3)]
    gen = ChunkedGenerator(9, cams, p3, p2, 4, pad=5, causal_shift=3, shuffle=True, random_seed=3, augment=True,
                           kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
    _, pairs = gen.next_pairs()
    n = len(pairs)
    assert n % 9 == 7
    table = torch.as_tensor(pairs.astype(np.int32)).cuda()
    batch = torch.zeros((), dtype=torch.int64, device='cuda')
    for b in range(gen.num_batches):
        rows = pairs[b * 9:(b + 1) * 9]
        want = P.chunk_gather(gen.seqs, rows, 4, 5, 3, LEFT, RIGHT, LEFT, RIGHT)
        batch.fill_(b)
        got = P.chunk_gather_indexed(gen.seqs, table, batch, len(rows), 9, 4, 5, 3, LEFT, RIGHT, LEFT, RIGHT)
        for w, g in zip(want, got):
            assert w.shape == g.shape and torch.equal(w, g), b
    assert any(r[3] for r in pairs) and any(not r[3] for r in pairs)


@pytest.mark.parametrize('amsgrad', [True, False])
@pytest.mark.parametrize('wd', [0.0, 0.01])
def test_indexed_adam_is_adam(amsgrad, wd):
    """6 steps, the lr changes between steps 3 and 4: parameters and all three moment buffers, bit for bit"""
    gen = torch.Generator().manual_seed(5)
    shapes = [(300, 70), (5000,), (17, 3)]
    init = [torch.randn(s, generator=gen) for s in shapes]
    grads = [[torch.randn(s, generator=gen) for s in shapes] for _ in range(6)]
    pa = [t.clone().cuda() for t in init]
    pb = [t.clone().cuda() for t in init]
    for p in pa + pb:
        p.requires_grad_(True)
        p.grad = torch.zeros_like(p)
    oa = P.FusedAdam(pa, lr=2e-3, amsgrad=amsgrad, weight_decay=wd)
    ob = P.FusedAdam(pb, lr=2e-3, amsgrad=amsgrad, weight_decay=wd)
    batch = torch.zeros((), dtype=torch.int64, device='cuda')
    for half, lr in ((0, 2e-3), (1, 7e-4)):
        oa.param_groups[0]['lr'] = ob.param_groups[0]['lr'] = lr
        coef = torch.as_tensor(P.adam_step_table(lr, BETAS, ob.step_count + 1, 3)).cuda()
        batch.zero_()
        for s in range(3):
            for p, q, g in zip(pa, pb, grads[3 * half + s]):
                p.grad.copy_(g)
                q.grad.copy_(g)
            oa.step()
            ob.step_indexed(coef, batch)
            batch += 1
        ob.step_count += 3
    assert oa.step_count == ob.step_count == 6
    for p, q in zip(pa, pb):
        assert torch.equal(p, q)
    for k in ('exp_avg', 'exp_avg_sq', 'max_exp_avg_sq'):
        a, b = getattr(oa, k), getattr(ob, k)
        assert (a is None) == (b is None) == (not amsgrad and k == 'max_exp_avg_sq')
        if a is not None:
            assert torch.equal(a, b), k


# ---------------------------------------------------------------------------------------------------------------
@needs_callers
@pytest.mark.parametrize('tprec', ['fp32', 'tf32'])
@pytest.mark.parametrize('name', list(MODELS))
def test_epochs_equal_main_train(callers, name, core, tprec):
    """two epochs with an lr decay between them: EpochTrainer against main.train over the device generator and over
    the reference's host generator (same seed), each with FusedAdam: parameters, BatchNorm statistics and
    num_batches_tracked, Adam moments and step_count, and the epoch losses as Python floats"""
    rec, mn = callers
    kind, ch, chunk, B = MODELS[name]
    p2, p3 = _split(3, LENGTHS, 7)
    make = lambda: engine.set_training_precision(_model(kind, ch), tprec)  # noqa: E731
    mt, md, mh = make(), make(), make()
    gt = _dgen(p2, p3, chunk, B)
    gd = _dgen(p2, p3, chunk, B)
    gh = rec.ChunkedGenerator(B, None, p3, p2, chunk, pad=13, causal_shift=0, shuffle=True, random_seed=1234,
                              augment=True, kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
    assert gt.num_batches * B > len(gt.pairs) > (gt.num_batches - 1) * B
    ot, od, oh = _adam(mt), _adam(md), _adam(mh)
    tr = training.EpochTrainer(mt, gt, ot)
    for epoch in range(2):
        lt = tr.train_epoch()
        ld = epochref.main_train_device(mn, md, gd, od)
        lh = mn.train(mh, gh, oh)
        assert isinstance(lt, float) and lt == ld == lh, (epoch, lt, ld, lh)
        st = _state(mt, ot)
        _assert_same(st, _state(md, od))
        _assert_same(st, _state(mh, oh))
        for o in (ot, od, oh):
            _decay(o)
    assert ot.step_count == 2 * gt.num_batches
    bn = [mod for mod in mt.modules() if isinstance(mod, torch.nn.BatchNorm2d)]
    assert bn and all(int(mod.num_batches_tracked) == 2 * gt.num_batches for mod in bn)


# ---------------------------------------------------------------------------------------------------------------
def _dropout_trainer(drop, lr):
    m = _model('o1f', 32, drop=drop)
    p2, p3 = _split(3, LENGTHS, 7)
    from device.common.generators import ChunkedGenerator
    gen = ChunkedGenerator(sum(LENGTHS), None, p3, p2, 1, pad=13, shuffle=False, augment=False)
    assert gen.num_batches == 1
    opt = _adam(m, lr=lr)
    return training.EpochTrainer(m, gen, opt), m, opt


def test_dropout_masks_repeat_and_move():
    """one batch per epoch, no shuffle, lr 0: the parameters never change and the forward in train mode reads no
    running statistic, so an epoch's loss depends on the dropout masks alone.  Without dropout every epoch gives the
    same loss; with it, no two consecutive epochs (steps) do, and two runs from the same state and counter agree."""
    tr0, _, _ = _dropout_trainer(0.0, 0.0)
    l0 = [tr0.train_epoch() for _ in range(4)]
    assert len(set(l0)) == 1, l0
    tr, m, opt = _dropout_trainer(0.25, 0.0)
    ds = m.__dict__['_gast_dropout_state']
    c0 = int(ds)
    sd, st = copy.deepcopy(m.state_dict()), copy.deepcopy(opt.state_dict())
    runs = []
    for _ in range(2):
        m.load_state_dict(sd)
        opt.load_state_dict(st)
        ds.fill_(c0)
        runs.append([tr.train_epoch() for _ in range(4)])
        step = 0xD1B54A32D192ED03
        want = (c0 + 4 * step) % (1 << 64)
        assert int(ds) % (1 << 64) == want
    assert runs[0] == runs[1]
    assert all(a != b for a, b in zip(runs[0], runs[0][1:])), runs[0]
    assert runs[0][0] != l0[0]


def test_epoch_makes_no_host_round_trip():
    m = _model('o1f', 32)
    p2, p3 = _split(3, LENGTHS, 7)
    gen = _dgen(p2, p3, 1, 40)
    tr = training.EpochTrainer(m, gen, _adam(m))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        s, losses = tr.train_epoch_async()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert losses.shape == (gen.num_batches,) and losses.dtype == torch.float32 and s.dtype == torch.float64
    w = torch.tensor([40] * (gen.num_batches - 1) + [len(gen.pairs) - 40 * (gen.num_batches - 1)], dtype=torch.float64)
    assert torch.isfinite(losses).all() and float(s) == float((w * losses.double().cpu()).cumsum(0)[-1])


def test_construction_leaves_no_trace():
    """the full state dict, the moments, step_count, the dropout counter and torch's RNG, byte for byte"""
    m = _model('o1f', 32, drop=0.25)
    p2, p3 = _split(3, LENGTHS, 7)
    gen = _dgen(p2, p3, 1, 40)
    opt = _adam(m)
    m.__dict__['_gast_dropout_state'] = torch.full((1,), 12345, dtype=torch.int64, device='cuda')
    for p in opt.params:                                        # non-zero moments and step count
        p.grad = torch.randn_like(p)
    opt.step()
    before = _state(m, opt)
    ds = m.__dict__['_gast_dropout_state'].clone()
    rng = torch.get_rng_state()
    rs = copy.deepcopy(gen.random_state().get_state())
    training.EpochTrainer(m, gen, opt)
    torch.cuda.synchronize()
    _assert_same(before, _state(m, opt))
    assert torch.equal(ds, m.__dict__['_gast_dropout_state'])
    assert torch.equal(rng, torch.get_rng_state())
    after = gen.random_state().get_state()
    assert all(np.array_equal(a, b) if isinstance(a, np.ndarray) else a == b for a, b in zip(rs, after))
    assert '_gast_direct_grads' not in m.__dict__


@needs_callers
def test_eval_epoch_is_main_eval(callers):
    rec, mn = callers
    m = _model('o1f', 32)
    p2, p3 = _split(3, LENGTHS, 7)
    tr = training.EpochTrainer(m, _dgen(p2, p3, 1, 40), _adam(m))
    tr.train_epoch()
    t2, t3 = _split(4, [60, 45, 33, 80], 9)
    mp_ref = _model('dilated', 32)
    mp = _model('dilated', 32)
    got = tr.eval_epoch(mp, t2, t3, p2, p3)
    test_gen = rec.UnchunkedGenerator(None, t3, t2, pad=13, causal_shift=0, augment=False, kps_left=LEFT,
                                      kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
    train_gen = rec.UnchunkedGenerator(None, p3, p2, pad=13, causal_shift=0, augment=False)
    want = mn.eval(m.state_dict(), mp_ref, test_gen, train_gen)
    assert not mp.training
    for g, w in zip(got, want):
        assert abs(g - w) <= 1e-6 * abs(w), (got, want)
    # zero-length sequences are skipped
    e2 = [np.zeros((0, 17, 2), np.float32)]
    e3 = [np.zeros((0, 17, 3), np.float32)]
    assert tr.eval_epoch(mp, t2 + e2, t3 + e3, e2 + p2, e3 + p3) == got


def test_resume_equals_uninterrupted():
    """checkpoint after epoch 1 (and trainval's lr decay), through torch.save / torch.load, into a fresh trainer"""
    p2, p3 = _split(3, LENGTHS, 7)
    m = _model('dilated', 32)
    gen, opt = _dgen(p2, p3, 4, 12), _adam(m)
    tr = training.EpochTrainer(m, gen, opt)
    tr.train_epoch()
    _decay(opt)
    buf = io.BytesIO()
    torch.save(tr.checkpoint(), buf)
    l2 = tr.train_epoch()
    want = _state(m, opt)
    buf.seek(0)
    chk = torch.load(buf, weights_only=False)
    assert chk['epoch'] == 1 and chk['lr'] == 1e-3 * DECAY and set(chk) == {'epoch', 'lr', 'random_state', 'optimizer',
                                                                            'model_pos'}
    m2 = _model('dilated', 32, seed=9)                           # other weights: all of them come from the checkpoint
    opt2 = _adam(m2)
    tr2 = training.EpochTrainer(m2, _dgen(p2, p3, 4, 12, seed=1), opt2, checkpoint=chk)
    assert tr2.epoch == 1 and opt2.param_groups[0]['lr'] == chk['lr']
    assert tr2.train_epoch() == l2 and tr2.epoch == 2
    _assert_same(want, _state(m2, opt2))


def test_refusals_before_any_launch(monkeypatch):
    p2, p3 = _split(3, LENGTHS, 7)

    def check(m, gen, opt, match):
        sd = {k: v.clone() for k, v in m.state_dict().items()}
        with pytest.raises(GastError, match=match):
            training.EpochTrainer(m, gen, opt)
        _assert_same(sd, {k: v for k, v in m.state_dict().items()})
        assert all(p.grad is None for p in m.parameters()) and '_gast_dropout_state' not in m.__dict__
    m = _model('o1f', 32)
    gen = _dgen(p2, p3, 1, 40)
    check(m, gen, P.FusedAdam(list(m.parameters())[1:], lr=1e-3, amsgrad=True), 'FusedAdam over exactly')
    check(m, gen, torch.optim.Adam(m.parameters(), lr=1e-3, amsgrad=True), 'FusedAdam over exactly')
    check(m, _dgen(p2, p3, 1, 40, endless=True), _adam(m), 'not endless')
    check(m, _dgen(p2, p3, 4, 12), _adam(m), 'chunk length 1')
    check(m.eval(), gen, _adam(m), 'eval mode')
    m.train()
    engine.set_precision(m, 'tf32')
    check(m, gen, _adam(m), 'inference-only')
    engine.set_precision(m, 'fp32')
    mh = _model('o1f', 32).half()
    check(mh, gen, None, 'half precision')
    monkeypatch.setattr(torch.distributed, 'is_initialized', lambda: True)
    monkeypatch.setattr(torch.distributed, 'get_world_size', lambda group=None: 2)
    check(m, gen, _adam(m), 'world size 2')
