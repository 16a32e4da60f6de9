"""The kink-free test points of tests/kinkfree.py, on the CPU: every ReLU and LeakyReLU input keeps its distance
from the kink, and the fp32 torch-CPU port meets the per-tensor gradient bars of tests/test_gpu_grad_exact.py
against its own fp64 run there.  This shows that fp32 arithmetic can reach those bars, and keeps the construction
honest when the port changes."""
import pytest
import torch

import kinkfree as K


@pytest.mark.parametrize('name', sorted(K.CASES))
def test_kink_free_point_and_fp32_port_bars(name):
    case = K.CASES[name]
    ref = K.reference(name)
    relu, leaky, per = ref['margins']
    assert relu >= K.MARGIN and leaky >= K.MARGIN, (relu, leaky, sorted(per.items(), key=lambda t: t[1])[:4])
    # the construction keeps both sides of every kink in use: no gradient tensor is zeroed wholesale, except the
    # bias of the input BatchNorm in train mode (the batch-statistics expand BatchNorm removes any constant it adds)
    zero = {k for k, (l2, _) in K.errors(ref['grads'], ref['grads'], ref['scales']).items() if l2 is None}
    assert zero == ({'init_bn.bias'} if case.training else set()), zero
    y, loss, g32, _ = K.port_grads(ref['sd'], ref['x'], ref['target'], case, torch.float32)
    assert (y - ref['y']).abs().max().item() <= K.Y_BAR * ref['y'].abs().max().item()
    assert abs(loss - ref['loss']) <= K.LOSS_BAR * abs(ref['loss'])
    bad, err = K.check(g32, ref['grads'], ref['scales'], 'ffma')
    assert not bad, bad


def test_observer_leaves_the_port_unchanged():
    """the kink observer sees every ReLU and LeakyReLU input in forward order and changes no bit of the result"""
    case = K.CASES['causal_T40_j19_c16_eval']
    sd = K.module(case).state_dict()
    x = K.inputs(case)
    seen = []
    y0 = K.port_forward(sd, x, case)
    y1 = K.port_forward(sd, x, case, tap=lambda name, h: seen.append(name))
    assert torch.equal(y0, y1)
    heads = [k for k in seen if k.endswith('.attentions.0.')]
    assert seen[:2] == ['expand_bn.', 'layers_graph_conv.0.local_graph_layer.bn_1.'] and len(heads) == 3
    assert len(seen) == 1 + 3 * (5 + 4) + 2 * 2
