"""Gradient goldens: run the UNMODIFIED reference (as tests/golden/make_golden.py does, whose set-up and helpers this
script reuses) on CPU fp32 with x.requires_grad_() and `loss = mpjpe(model(x), target)` (common/loss.py:5-11).

    python tests/golden/make_golden_grad.py

Writes tests/golden/grad_*.npz: x, target, y, loss and dL/dx; per parameter the fingerprint make_golden.py:train_case
stores (norm, sum, 48 largest entries; the whole gradient for the small cases); the reference's own 8-vs-3-thread
spread as alt_*.  Weights are re-created from `gast_b200.synth`, as for every golden.
"""
import numpy as np
import torch

from make_golden import SpatioTemporalModel, SpatioTemporalModelOptimized1f, adj_for, save, _digest, synth


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
    with torch.enable_grad():
        y = m(x)
        tgt = torch.from_numpy((0.5 * np.random.RandomState(meta['xseed'] + 1).standard_normal(tuple(y.shape)))
                               .astype(np.float32))
        loss = mpjpe(y, tgt)
        loss.backward()
    grads = {k: prm.grad.detach().clone() for k, prm in m.named_parameters()}
    return m, dict(x=x.detach().numpy().copy(), target=tgt.numpy().copy(), y=y.detach().contiguous().numpy().copy(),
                   loss=loss.item(), dx=x.grad.numpy().copy(), grads=grads)


def grad_case(name, J, fw, ch, B, T, strided, training, full_grads, causal=False, dropout=0.25, seed=9, xseed=300):
    """Gradients of the reference with respect to its parameters AND its input, in eval() mode (BatchNorm on the
    running statistics, Dropout off: the module's `dropout` must not matter) or in train() mode (dropout 0)."""
    meta = dict(kind='grad', J=J, filter_widths=fw, channels=ch, B=B, T=T, strided=strided, causal=causal, dense=False,
                training=training, dropout=0.0 if training else dropout, seed=seed, xseed=xseed, full_grads=full_grads,
                threads=8, alt_threads=3)
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
    save(name, meta=meta, **out)
    print('   reference self-noise (8 vs 3 threads): loss rel %.3g, grad rel L2 %.3g, dx rel L2 %.3g'
          % (abs(out['alt_loss0'] - out['loss0']) / out['loss0'], out['alt_dg0'], out['alt_dx']))


def main():
    # whole gradients where they stay small (the 19-joint two-stage and the 16-channel models); the 17-joint
    # 32-channel cases keep the fingerprints only, which the training goldens show are enough to pin every tensor
    grad_case('grad_eval_17_333_c32_b6', 17, [3, 3, 3], 32, 6, 27, strided=True, training=False, full_grads=False)
    grad_case('grad_eval_19_33_c32_b5', 19, [3, 3], 32, 5, 9, strided=True, training=False, full_grads=True)
    grad_case('grad_eval_17_333_c16_causal_dilated_T40', 17, [3, 3, 3], 16, 2, 40, strided=False, training=False,
              full_grads=True, causal=True)
    grad_case('grad_eval_cfg3_17_333_c128_b32', 17, [3, 3, 3], 128, 32, 27, strided=True, training=False,
              full_grads=False)
    grad_case('grad_train_17_333_c32_b6', 17, [3, 3, 3], 32, 6, 27, strided=True, training=True, full_grads=False)


if __name__ == '__main__':
    main()
