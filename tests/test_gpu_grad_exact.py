"""Every gradient tensor of the lifting network on the GPU, per tensor, against fp64 autograd of the torch-CPU port
at the kink-free test points of tests/kinkfree.py: y, the loss, every parameter gradient, dL/dx, and dL/dx of the
input-only path (every parameter frozen) in train mode (batch statistics, with and without dropout: the masks are
the library's own, replayed into the port by tests/dropoutref.py) and eval mode (running statistics), on both GEMM
cores.  No ReLU or LeakyReLU input lies near its kink there, so fp64 is an exact reference and every
tensor is held to a rounding-level bar: a fault confined to one small tensor (C_k, concat_project, e, a BatchNorm
bias, a tail column of a weight gradient, one split of a reduction) fails it."""
import os

import pytest
import torch

from gast_b200 import engine
import kinkfree as K

pytestmark = pytest.mark.gpu

REPORT_DIR = os.environ.get('GAST_TEST_REPORT_DIR')   # optional directory for the measured errors of these tests


@pytest.fixture(params=[0, 1], ids=['auto', 'ffma'])
def core(request):
    engine.set_gemm_core(request.param)
    yield request.param
    engine.set_gemm_core(0)


def _mpjpe(y, t):
    return torch.mean(torch.norm(y - t, dim=3))


def _run(case, ref, frozen):
    m = K.module(case)
    m.load_state_dict(ref['sd'])
    m = m.cuda().train(case.training).requires_grad_(not frozen)
    x = ref['x'].cuda().requires_grad_()
    torch.manual_seed(K.DROP_SEED)      # the dropout masks of the reference (kinkfree.drop_masks)
    y = m(x)
    loss = _mpjpe(y, ref['target'].cuda())
    loss.backward()
    got = {} if frozen else {k: p.grad.cpu().double() for k, p in m.named_parameters()}
    got['x'] = x.grad.cpu().double()
    if frozen:
        assert all(p.grad is None for p in m.parameters())
    return y.detach().cpu().double(), float(loss), got


def dense_tn_split(M, N, K_, sms):
    """(row splits, rows per split) of the weight-gradient contraction dense_tn (csrc/train.cuh) for M rows"""
    tiles = -(-N // 128) * -(-K_ // 128)
    S = max(1, min(-(-M // 256), -(-2 * sms // tiles)))
    rps = -(-(-(-M // S)) // 16) * 16
    return -(-M // rps), rps


def test_case_matrix_reaches_split_reductions():
    """the 128-channel train case splits the weight-gradient row contraction of its first block into several row
    ranges with a ragged last one, and semch_dcoef_kernel into several frame ranges"""
    case = K.CASES['o1f_j17_c128_train']
    F0 = case.B * (case.T // case.fw[0])
    M0 = F0 * case.J
    S, rps = dense_tn_split(M0, case.ch, case.ch, torch.cuda.get_device_properties(0).multi_processor_count)
    assert S > 1 and M0 % rps != 0, (M0, S, rps)
    assert max(1, min(32, F0 // 32)) > 1, F0


@pytest.mark.parametrize('name', sorted(K.CASES))
def test_every_gradient_vs_fp64_port(name, core):
    case = K.CASES[name]
    ref = K.reference(name)
    relu, leaky, _ = ref['margins']
    assert relu >= K.MARGIN and leaky >= K.MARGIN, (relu, leaky)
    y, loss, got = _run(case, ref, frozen=False)
    y_err = (y - ref['y']).abs().max().item() / ref['y'].abs().max().item()
    loss_err = abs(loss - ref['loss']) / abs(ref['loss'])
    bad, err = K.check(got, ref['grads'], ref['scales'], 'ffma' if core == 1 else 'tc')
    # the input-only path (every parameter frozen) gives the dL/dx of the full backward
    _, _, frozen = _run(case, ref, frozen=True)
    dx_diff = (frozen['x'] - got['x']).abs().max().item() / got['x'].abs().max().item()
    if REPORT_DIR:
        os.makedirs(REPORT_DIR, exist_ok=True)
        l2w = max((v for v in err.items() if v[1][0] is not None), key=lambda t: t[1][0])
        mxw = max((v for v in err.items() if v[1][0] is not None), key=lambda t: t[1][1])
        zero = max((v[1] for v in err.values() if v[0] is None), default=0.0)
        with open(os.path.join(REPORT_DIR, 'grad_exact.txt'), 'a') as f:
            f.write('%s core %d: y %.2e loss %.2e | worst l2 %.2e %s | worst max %.2e %s | dx l2 %.2e max %.2e | '
                    'zero %.1e | input-only dx %.1e | margins %.1e %.1e\n'
                    % (name, core, y_err, loss_err, l2w[1][0], l2w[0], mxw[1][1], mxw[0], err['x'][0], err['x'][1],
                       zero, dx_diff, relu, leaky))
    assert y_err <= K.Y_BAR, y_err
    assert loss_err <= K.LOSS_BAR, loss_err
    assert not bad, sorted(bad, key=lambda t: -(t[1] or 0))[:12]
    assert dx_diff <= 1e-6, dx_diff
