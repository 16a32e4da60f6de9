"""GPU: training in the TF32 training precision (engine.set_training_precision(model, 'tf32')) against the default
fp32-grade one, in one process: the card's name, power limit and SM clock (read before and after the timings), then
  * training steps (FusedAdam amsgrad, dropout 0.05) of the Optimized1f 27f/17j/128ch and 81f/17j/64ch models at
    b = 128 and 1024, eager (DataParallelTrainer) and graphed (GraphedTrainer), fp32 and TF32 alternated, three runs
    each (ms per step on the device stream, CUDA events after a warm-up of every shape);
  * the eval-mode backward of tools/train_step.py's `eval` shape (27f/128ch, b = 128: parameter gradients and dL/dx);
  * every weight-gradient contraction (dense_tn) of one b = 128 27f/128ch step on both weight-gradient kernels through
    gast_debug_wgrad.
`--profile DIR`: instead, one eager b = 128 27f/128ch step per mode under torch.profiler (CUDA activities), split
into GEMMs, weight gradients, BatchNorm, other kernels and the gaps between kernels; the traces go to DIR.
One JSON line per measurement.

    python tools/train_precision_bench.py [--steps K] [--profile DIR]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
from gast_b200 import _lib, engine, synth  # noqa: E402
from gast_b200.pipeline import FusedAdam  # noqa: E402
from gast_b200.trainer import DataParallelTrainer, GraphedTrainer  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f  # noqa: E402
from launch_times import card  # noqa: E402

J = 17
CONFIGS = {'27f_128ch': ([3, 3, 3], 128, 27), '81f_64ch': ([3, 3, 3, 3], 64, 81)}


def emit(d):
    print(json.dumps(d), flush=True)


def model(fw, ch, prec, dropout=0.05):
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=False, dropout=dropout, channels=ch)
    synth.randomize_module(m, 1)
    return engine.set_training_precision(m.cuda(), prec)


def trainer(cfg, b, prec, graphed):
    fw, ch, T = CONFIGS[cfg]
    m = model(fw, ch, prec)
    opt = lambda ps: FusedAdam(ps, lr=1e-4, amsgrad=True)   # noqa: E731
    tr = GraphedTrainer(m, opt, (b, T, J, 2), (b, 1, J, 3)) if graphed else DataParallelTrainer(m, opt)
    x = torch.from_numpy(synth.synth_input(b, T, J, 2, seed=3)).cuda()
    y = torch.from_numpy(synth.synth_target(b, J, seed=4)).cuda()
    return tr, x, y


def timed(fn, warm, reps):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def train_steps(steps):
    for cfg in CONFIGS:
        for b in (128, 1024):
            for graphed in (False, True):
                setups = {p: trainer(cfg, b, p, graphed) for p in ('fp32', 'tf32')}
                runs = {'fp32': [], 'tf32': []}
                for _ in range(3):
                    for p in ('fp32', 'tf32'):
                        tr, x, y = setups[p]
                        runs[p].append(timed(lambda: tr.step(x, y), 3, steps))
                d = {'what': 'train_step', 'config': cfg, 'b': b, 'graphed': graphed}
                for p in runs:
                    d[p + '_ms'] = [round(v, 4) for v in runs[p]]
                    d[p + '_median_ms'] = round(float(np.median(runs[p])), 4)
                    d[p + '_spread'] = round((max(runs[p]) - min(runs[p])) / float(np.median(runs[p])), 4)
                d['speedup'] = round(d['fp32_median_ms'] / d['tf32_median_ms'], 4)
                emit(d)
                del setups
                torch.cuda.empty_cache()


def eval_backward(steps):
    fw, ch, T = CONFIGS['27f_128ch']
    b = 128
    ms = {p: model(fw, ch, p).eval() for p in ('fp32', 'tf32')}
    x = torch.from_numpy(synth.synth_input(b, T, J, 2, seed=3)).cuda()
    y = torch.from_numpy(synth.synth_target(b, J, seed=4)).cuda()

    def fwd_bwd(m):
        xx = x.clone().requires_grad_()
        torch.mean(torch.norm(m(xx) - y, dim=3)).backward()

    runs = {'fp32': [], 'tf32': []}
    for _ in range(3):
        for p in runs:
            runs[p].append(timed(lambda: fwd_bwd(ms[p]), 3, steps))
    d = {'what': 'eval_backward', 'config': '27f_128ch', 'b': b}
    for p in runs:
        d[p + '_ms'] = [round(v, 4) for v in runs[p]]
        d[p + '_median_ms'] = round(float(np.median(runs[p])), 4)
    d['speedup'] = round(d['fp32_median_ms'] / d['tf32_median_ms'], 4)
    emit(d)


def step_shapes(C, fw, B, T):
    """(M, N, K) of every dense_tn of one training step of the Optimized1f model"""
    out = []
    F = B * (T // fw[0])
    out.append((F * J, C, -(-fw[0] * 2 // 8) * 8))
    for i in range(len(fw)):
        Cb = C << i
        if i:
            F //= fw[i]
            out += [(F * J, Cb, Cb), (F * J, Cb, fw[i] * Cb)]
        out += [(F * J, 2 * Cb, 3 * Cb), (F * J, Cb, Cb), (F * J, Cb, Cb), (F * J, 8, Cb), (F * J, Cb, 2 * Cb),
                (F * J, 4 * Cb, Cb)]
    return out


def wgrad_contractions():
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    tot = {'ffma': 0.0, 'tf32': 0.0}
    import ctypes as C
    for (M, N, K) in step_shapes(128, [3, 3, 3], 128, 27):
        dz = torch.randn(M, N, device='cuda')
        a = torch.randn(M, K, device='cuda').abs()
        out = torch.empty(N, K, device='cuda')
        d = {'what': 'wgrad', 'M': M, 'N': N, 'K': K}
        for name, core, mode in (('ffma', 1, 0), ('tf32', 0, 1)):
            ms = C.c_float(0.0)
            rc = lib.gast_debug_wgrad(dz.data_ptr(), a.data_ptr(), out.data_ptr(), M, N, K, core, mode, 50,
                                      C.byref(ms), st)
            if rc != 0:
                raise RuntimeError(_lib.last_error())
            d[name + '_ms'] = round(ms.value, 5)
            tot[name] += ms.value
        d['tf32_kernel'] = N % 32 == 0 and K % 32 == 0
        emit(d)
    emit({'what': 'wgrad_total_one_step', 'config': '27f_128ch', 'b': 128, 'ffma_ms': round(tot['ffma'], 4),
          'tf32_ms': round(tot['tf32'], 4)})


def classify(name):
    if 'wgrad' in name:
        return 'weight_gradients'
    if 'gemm_tc_kernel' in name or 'gemm_ffma_kernel' in name:
        return 'gemms'
    if 'bn_' in name or 'col_stats' in name:
        return 'batchnorm'
    return 'other'


def profile(out_dir):
    from torch.profiler import profile as tprofile, ProfilerActivity
    os.makedirs(out_dir, exist_ok=True)
    fw, ch, T = CONFIGS['27f_128ch']
    for p in ('fp32', 'tf32'):
        tr, x, y = trainer('27f_128ch', 128, p, False)
        for _ in range(5):
            tr.step(x, y)
        torch.cuda.synchronize()
        with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
            tr.step(x, y)
            torch.cuda.synchronize()
        prof.export_chrome_trace(os.path.join(out_dir, 'train_step_%s.json' % p))
        ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        ev.sort(key=lambda e: e.time_range.start)
        split = {'gemms': 0.0, 'weight_gradients': 0.0, 'batchnorm': 0.0, 'other': 0.0}
        count = {k: 0 for k in split}
        busy, end = 0.0, None
        for e in ev:
            k = classify(e.name)
            dur = (e.time_range.end - e.time_range.start) / 1e3
            split[k] += dur
            count[k] += 1
            s, t = e.time_range.start, e.time_range.end
            if end is None or s >= end:
                busy += (t - s) / 1e3
                end = t
            elif t > end:
                busy += (t - end) / 1e3
                end = t
        span = (ev[-1].time_range.end - ev[0].time_range.start) / 1e3 if ev else 0.0
        d = {'what': 'profile_eager_step', 'precision': p, 'config': '27f_128ch', 'b': 128,
             'span_ms': round(span, 4), 'gaps_ms': round(span - busy, 4)}
        for k in split:
            d[k + '_ms'] = round(split[k], 4)
            d[k + '_kernels'] = count[k]
        emit(d)
        del tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--profile', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('train_precision_bench: no CUDA device')
    emit(dict(card(), what='card'))
    if a.profile:
        profile(a.profile)
    else:
        train_steps(a.steps)
        eval_backward(a.steps)
        wgrad_contractions()
    emit(dict(card(), what='card_after'))


if __name__ == '__main__':
    main()
