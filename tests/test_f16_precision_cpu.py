"""The fp16 inference precision on the host: engine.set_precision takes 'fp16' and get_precision returns it, the
training precision does not, and a stream pool's ring storage follows the precision (PoseStream._alloc_state) without
any device work until a call needs the state."""
import pytest

from gast_b200 import engine, synth


def _model():
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    return SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], channels=32).eval()


def test_set_precision_takes_fp16():
    m = _model()
    assert engine.set_precision(m, 'fp16') is m
    assert all(engine.get_precision(s) == 'fp16' for s in m.modules())
    assert engine.get_training_precision(m) == 'fp32'
    engine.set_precision(m, 'fp32')
    assert engine.get_precision(m) == 'fp32'


@pytest.mark.parametrize('mode', ['FP16', 'half', 16])
def test_set_precision_names_fp16_in_its_refusal(mode):
    with pytest.raises(engine.GastError, match="'fp16'"):
        engine.set_precision(_model(), mode)


def test_training_precision_refuses_fp16():
    m = _model()
    with pytest.raises(engine.GastError, match="'fp32' or 'tf32'"):
        engine.set_training_precision(m, 'fp16')
    assert engine.get_training_precision(m) == 'fp32'


def test_fp32_only_names_the_mode():
    m = _model()
    engine.set_precision(m, 'fp16')
    with pytest.raises(engine.GastError, match=r"fp16 precision, which is inference-only.*set_precision\(model, 'fp32'\)"):
        engine._fp32_only(m, 'forward')
    engine.set_precision(m, 'tf32')
    with pytest.raises(engine.GastError, match=r"TF32, which is inference-only"):
        engine._fp32_only(m, 'forward')
    engine.set_training_precision(m, 'tf32')
    engine._fp32_only(m, 'forward')
    engine.set_precision(m, 'fp16')
    engine._fp32_only(m, 'forward')
