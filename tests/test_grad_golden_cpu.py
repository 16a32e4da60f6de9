"""Gradients of the lifting network with respect to its parameters and its 2D input, in eval() mode (BatchNorm on the
running statistics, Dropout off) and in train() mode: the differentiable torch-CPU port (oracle/gast_torch_ref.py)
against fixtures of the UNMODIFIED reference (tests/golden/grad_*.npz, make_golden_grad.py).  A train-mode fixture
with dropout stores the masks it ran with (the library's own, tests/dropoutref.py); the port applies them too.  This
pins the oracle the GPU tests of tests/test_gpu_eval_grad.py compare against.  CPU only."""
import numpy as np
import pytest
import torch

from conftest import load_golden, golden_names
from oracle import gast_oracle as O
from gast_b200 import synth
import dropoutref as D
import train_fixture as TF


def grad_module(meta):
    """our drop-in module shell with the fixture's weights and running statistics (synth is keyed on state_dict
    names, so these are the ones the reference model had)"""
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    J, fw = meta['J'], meta['filter_widths']
    if meta['strided']:
        m = SpatioTemporalModelOptimized1f(TF.adj_t(J), J, 2, J, fw, causal=meta['causal'], dropout=meta['dropout'],
                                           channels=meta['channels'])
    else:
        m = SpatioTemporalModel(TF.adj_t(J), J, 2, J, fw, causal=meta['causal'], dropout=meta['dropout'],
                                channels=meta['channels'], dense=meta['dense'])
    synth.randomize_module(m, meta['seed'])
    assert [k for k, _ in m.named_parameters()] == meta['names']
    return m.train(meta['training'])


def check_dx(g, dx, rtol, report=None):
    """dL/dx against the fixture: relative L2 error and largest entry error relative to max|dx|, both below rtol
    (or 3x the reference's own 8-vs-3-thread spread, whichever is larger)"""
    ref = g['dx']
    tol = max(rtol, 3.0 * float(g['alt_dx']))
    l2 = float(np.linalg.norm(dx - ref) / np.linalg.norm(ref))
    mx = float(np.abs(dx - ref).max() / np.abs(ref).max())
    if report is not None:
        report.append('dx: rel L2 %.3g, max %.3g (tolerance %.3g)' % (l2, mx, tol))
    return [] if (l2 < tol and mx < tol) else [('dx', l2, mx, tol)]


@pytest.mark.parametrize('name', golden_names('grad_'))
def test_torch_ref_gradients_match_reference_fixture(name):
    from oracle import gast_torch_ref as TR
    g = load_golden(name)
    meta = g['meta']
    m = grad_module(meta)
    p = {k: v.clone().requires_grad_(v.dtype.is_floating_point and 'running' not in k)
         for k, v in m.state_dict().items()}
    masks = tuple(torch.from_numpy(a) for a in O.local_masks(O.adj_from_parents(synth.skeleton_parents(meta['J']))))
    x = torch.from_numpy(g['x']).requires_grad_()
    drop = D.dropper(D.golden_masks(g)) if meta.get('drop_seed') is not None else 0.0
    threads = torch.get_num_threads()
    torch.set_num_threads(meta['threads'])      # the fixture's CPU summation order (make_golden_grad.py)
    try:
        y = TR.forward(x, p, masks, meta['filter_widths'], causal=meta['causal'], strided=meta['strided'],
                       training=meta['training'], stats={} if meta['training'] else None, drop=drop)
        loss = TR.mpjpe(y, torch.from_numpy(g['target']))
        loss.backward()
    finally:
        torch.set_num_threads(threads)
    bad = TF.check_step(g, 0, y.detach().numpy(), loss.item(), {k: p[k].grad for k in meta['names']},
                        y_tol=2e-6, loss_rtol=1e-6, ent_rtol=2e-3, norm_rtol=2e-3)
    bad += check_dx(g, x.grad.numpy(), 2e-3)
    if meta['full_grads']:
        for k in meta['names']:
            gr = g['grad0/' + k]
            if np.abs(gr).max() > 1e-12 and not np.abs(p[k].grad.numpy() - gr).max() <= 2e-3 * np.abs(gr).max():
                bad.append(('full gradient', k))
    assert not bad, bad[:10]
