"""Gradient goldens: run the UNMODIFIED reference (as tests/golden/make_golden.py does, whose set-up and helpers this
script reuses) on CPU fp32 with x.requires_grad_() and `loss = mpjpe(model(x), target)` (common/loss.py:5-11).

    python tests/golden/make_golden_grad.py

Writes tests/golden/grad_*.npz: x, target, y, loss and dL/dx; per parameter the fingerprint make_golden.py:train_case
stores (norm, sum, 48 largest entries; the whole gradient for the small cases); the reference's own 8-vs-3-thread
spread as alt_*.  Weights are re-created from `gast_b200.synth`, as for every golden.

A train-mode case with dropout (`drop_seed` in its meta) runs the reference with the masks the library draws in a
forward right after torch.manual_seed(drop_seed) (tests/dropoutref.py), applied in place of its own
torch.nn.functional.dropout, and stores them (keep/<site>, packed bits in (b, t, j, c) order).

    python tests/golden/make_golden_grad.py [name ...]      (only the named cases; all by default)
"""
import contextlib
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

from make_golden import SpatioTemporalModel, SpatioTemporalModelOptimized1f, adj_for, save, _digest, synth

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dropoutref as D  # noqa: E402


@contextlib.contextmanager
def _replayed_dropout(masks):
    """torch.nn.functional.dropout applies `masks` (site -> scaled mask) in site order; exactly one call per site"""
    order = list(masks.values())
    calls = []
    real = F.dropout

    def dropout(input, p=0.5, training=True, inplace=False):
        assert training and len(calls) < len(order), (training, len(calls))
        m = order[len(calls)]
        assert tuple(m.shape) == tuple(input.shape), (len(calls), tuple(m.shape), tuple(input.shape))
        calls.append(p)
        return input * m.to(input.dtype)
    F.dropout = dropout
    try:
        yield
    finally:
        F.dropout = real
    assert len(calls) == len(order), (len(calls), len(order))


def _grad_run(meta, threads):
    """`loss = mpjpe(model(x), target)` with x.requires_grad_(), one backward, no optimiser step"""
    from common.loss import mpjpe
    torch.set_num_threads(threads)
    J, fw, ch = meta['J'], meta['filter_widths'], meta['channels']
    adj = adj_for(J)
    if meta['strided']:
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=meta['causal'], dropout=meta['dropout'], channels=ch)
    else:
        m = SpatioTemporalModel(adj, J, 2, J, fw, causal=meta['causal'], dropout=meta['dropout'], channels=ch)
    synth.randomize_module(m, meta['seed'])
    m.train(meta['training'])
    x = torch.from_numpy(synth.synth_input(meta['B'], meta['T'], J, 2, seed=meta['xseed'])).requires_grad_()
    replay = contextlib.nullcontext()
    if meta.get('drop_seed') is not None:
        replay = _replayed_dropout(D.masks(meta, meta['B'], meta['T'], J, meta['dropout'],
                                           D.engine_seed(meta['drop_seed'])))
    with torch.enable_grad():
        with replay:
            y = m(x)
        tgt = torch.from_numpy((0.5 * np.random.RandomState(meta['xseed'] + 1).standard_normal(tuple(y.shape)))
                               .astype(np.float32))
        loss = mpjpe(y, tgt)
        loss.backward()
    grads = {k: prm.grad.detach().clone() for k, prm in m.named_parameters()}
    return m, dict(x=x.detach().numpy().copy(), target=tgt.numpy().copy(), y=y.detach().contiguous().numpy().copy(),
                   loss=loss.item(), dx=x.grad.numpy().copy(), grads=grads)


def grad_case(name, J, fw, ch, B, T, strided, training, full_grads, causal=False, dropout=0.25, seed=9, xseed=300,
              drop_seed=None):
    """Gradients of the reference with respect to its parameters AND its input, in eval() mode (BatchNorm on the
    running statistics, Dropout off: the module's `dropout` must not matter) or in train() mode: dropout 0, or with
    `drop_seed` the library's masks of probability `dropout` (see the module's docstring)."""
    meta = dict(kind='grad', J=J, filter_widths=fw, channels=ch, B=B, T=T, strided=strided, causal=causal, dense=False,
                training=training, dropout=0.0 if (training and drop_seed is None) else dropout, seed=seed,
                xseed=xseed, full_grads=full_grads, threads=8, alt_threads=3)
    if drop_seed is not None:
        assert training
        meta['drop_seed'] = drop_seed
    m, r = _grad_run(meta, 8)
    _, a = _grad_run(meta, 3)
    torch.set_num_threads(8)
    names = [k for k, _ in m.named_parameters()]
    meta['names'] = names
    out = dict(x=r['x'], target=r['target'], y0=r['y'], loss0=np.array(r['loss'], np.float64), dx=r['dx'])
    for k in names:
        g = r['grads'][k].reshape(-1)
        idx = torch.topk(g.abs(), min(48, g.numel())).indices.sort().values
        out['idx/' + k] = idx.numpy().astype(np.int64)
        out['gsum0/' + k], out['gent0/' + k] = _digest(r['grads'][k], idx)
        if full_grads:
            out['grad0/' + k] = r['grads'][k].numpy().copy()
    out['alt_loss0'] = np.array(a['loss'], np.float64)
    out['alt_dy0'] = np.array(np.abs(a['y'] - r['y']).max(), np.float64)
    out['alt_dp0'] = np.array(0.0, np.float64)                  # no optimiser step
    out['alt_dg0'] = np.array(max(float((a['grads'][k] - r['grads'][k]).norm() / (r['grads'][k].norm() + 1e-30))
                                  for k in names if float(r['grads'][k].norm()) > 1e-5), np.float64)
    out['alt_dx'] = np.array(np.linalg.norm(a['dx'] - r['dx']) / np.linalg.norm(r['dx']), np.float64)
    if drop_seed is not None:
        packed = D.pack(D.masks(meta, B, T, J, dropout, D.engine_seed(drop_seed)))
        out.update(('keep/' + k, v) for k, v in packed.items())
    save(name, meta=meta, **out)
    print('   reference self-noise (8 vs 3 threads): loss rel %.3g, grad rel L2 %.3g, dx rel L2 %.3g'
          % (abs(out['alt_loss0'] - out['loss0']) / out['loss0'], out['alt_dg0'], out['alt_dx']))


def main(names=()):
    """every case, or only those in `names`"""
    def case(name, *a, **k):
        if not names or name in names:
            grad_case(name, *a, **k)
    # whole gradients where they stay small (the 19-joint two-stage and the 16-channel models); the 17-joint
    # 32-channel cases keep the fingerprints only, which the training goldens show are enough to pin every tensor
    case('grad_eval_17_333_c32_b6', 17, [3, 3, 3], 32, 6, 27, strided=True, training=False, full_grads=False)
    case('grad_eval_19_33_c32_b5', 19, [3, 3], 32, 5, 9, strided=True, training=False, full_grads=True)
    case('grad_eval_17_333_c16_causal_dilated_T40', 17, [3, 3, 3], 16, 2, 40, strided=False, training=False,
         full_grads=True, causal=True)
    case('grad_eval_cfg3_17_333_c128_b32', 17, [3, 3, 3], 128, 32, 27, strided=True, training=False, full_grads=False)
    case('grad_train_17_333_c32_b6', 17, [3, 3, 3], 32, 6, 27, strided=True, training=True, full_grads=False)
    # the library's own dropout masks at p = 0.25: pins the device's masks and their backward to the reference
    case('grad_train_drop25_17_333_c32_b6', 17, [3, 3, 3], 32, 6, 27, strided=True, training=True, full_grads=False,
         dropout=0.25, drop_seed=23)


if __name__ == '__main__':
    main(sys.argv[1:])
