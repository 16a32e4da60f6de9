"""Host-side checks of whole-epoch training (gast_b200.training.EpochTrainer): the Adam coefficient table is
gast_adam_step's own host arithmetic, and every refusal that needs no device comes before anything else is done."""
import math

import numpy as np
import pytest
import torch

from gast_b200 import engine, synth, training
from gast_b200 import pipeline as P
from gast_b200.engine import GastError


@pytest.mark.parametrize('lr,betas,first', [(1e-3, (0.9, 0.999), 1), (1e-3 * 0.95 ** 7, (0.9, 0.999), 4001),
                                            (3e-4, (0.8, 0.99), 17)])
def test_adam_table_is_adam_step_arithmetic(lr, betas, first):
    """{lr / bc1, sqrt(bc2)} in double with C pow, rounded to float (gast_adam_step, csrc/pipeline.cuh adam_coefs);
    Python's float ** is C pow"""
    n = 300
    got = P.adam_step_table(lr, betas, first, n)
    assert got.shape == (n, 2) and got.dtype == np.float32
    for i in range(n):
        s = first + i
        want = (np.float32(lr / (1.0 - betas[0] ** float(s))), np.float32(math.sqrt(1.0 - betas[1] ** float(s))))
        assert got[i, 0].tobytes() == want[0].tobytes() and got[i, 1].tobytes() == want[1].tobytes(), s


def test_adam_table_refuses_bad_steps():
    with pytest.raises(GastError, match='gast_adam_step_table'):
        P.adam_step_table(1e-3, (0.9, 0.999), 0, 4)
    with pytest.raises(GastError, match='gast_adam_step_table'):
        P.adam_step_table(1e-3, (0.9, 0.999), 1, 0)


def _model(**kw):
    from model.gast_net import SpatioTemporalModelOptimized1f
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    m = SpatioTemporalModelOptimized1f(adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], [])), 17, 2, 17,
                                       [3, 3, 3], channels=32, **kw)
    synth.randomize_module(m, 2)
    return m.train()


def _refused(m, opt, match, gen=None):
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(GastError, match=match):
        training.EpochTrainer(m, gen, opt)
    after = m.state_dict()
    assert all(torch.equal(sd[k], after[k]) for k in sd)
    assert all(p.grad is None for p in m.parameters()) and '_gast_dropout_state' not in m.__dict__


def test_refusals(monkeypatch):
    m = _model()
    adam = torch.optim.Adam(m.parameters(), lr=1e-3, amsgrad=True)
    _refused(m, adam, 'FusedAdam over exactly')
    _refused(m.eval(), adam, 'eval mode')
    m.train()
    engine.set_precision(m, 'fp16')
    _refused(m, adam, 'inference-only')
    engine.set_precision(m, 'fp32')
    _refused(_model().half(), adam, 'half precision')
    _refused(torch.nn.Linear(3, 3), adam, 'SpatioTemporalModel')
    monkeypatch.setattr(torch.distributed, 'is_initialized', lambda: True)
    monkeypatch.setattr(torch.distributed, 'get_world_size', lambda group=None: 4)
    _refused(m, adam, 'world size 4')
