"""engine.set_precision / get_precision on the host: the setting reaches every sub-module, is kept by deepcopy and by
nn.DataParallel's replicas (both copy the module's __dict__), stays out of state_dict, and refuses unknown modes."""
import copy

import pytest

from gast_b200 import engine, synth


def _model():
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    return SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], channels=32).eval()


def test_set_precision_reaches_sub_modules_and_copies():
    m = _model()
    keys = list(m.state_dict().keys())
    assert engine.get_precision(m) == 'fp32'
    assert engine.set_precision(m, 'tf32') is m
    assert all(engine.get_precision(s) == 'tf32' for s in m.modules())
    assert list(m.state_dict().keys()) == keys
    assert engine.get_precision(copy.deepcopy(m)) == 'tf32'
    rep = m._replicate_for_data_parallel()
    assert engine.get_precision(rep) == 'tf32'
    blk = m.layers_graph_conv[1]
    engine.set_precision(blk, 'fp32')
    assert engine.get_precision(blk) == 'fp32' and engine.get_precision(m) == 'tf32'
    engine.set_precision(m, 'fp32')
    assert all(engine.get_precision(s) == 'fp32' for s in m.modules())


@pytest.mark.parametrize('mode', ['bf16', 'TF32', 1, None])
def test_set_precision_refuses_unknown_modes(mode):
    with pytest.raises(engine.GastError, match='fp32'):
        engine.set_precision(_model(), mode)
