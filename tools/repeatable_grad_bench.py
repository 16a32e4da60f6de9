"""Cost of the fixed-order tap adjoints and column sums: training steps of two builds of the library, timed in one
session, one process per build and round, the builds alternated round by round (GAST_B200_LIB selects the library
each process loads).  Per build and round, after warm-up, CUDA events over --steps steps of:
  * the dilated SpatioTemporalModel 27f/128ch, b = 128, at T = 27 and T = 53 (graphed step: GraphedTrainer);
  * the dense ablation [3,3,3]/128ch, b = 128, T = 27 (graphed);
  * Optimized1f 27f/128ch, b = 128 (graphed, and eager as in tools/train_step.py);
each with dropout 0.25 (0.05 for Optimized1f, BASELINE configs[2]) and FusedAdam(amsgrad).  Each process also reports
the workspace queries at the shapes of DESIGN.md §11 and §11.1.  Prints one JSON line per process and a summary line
per case and build (median and range of the rounds); the first line has the card's name, power limit and SM clock.

    python tools/repeatable_grad_bench.py --lib new=PATH --lib parent=PATH [--rounds 3] [--steps 20] [--out FILE]

The eval-backward rows of DESIGN.md §11.1 are tools/chunked_grad_bench.py's, run once per build with GAST_B200_LIB set.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CASES = [  # name, model, T, dropout, graphed
    ('dilated_27f_128ch_b128_T27', 'dilated', 27, 0.25, True),
    ('dilated_27f_128ch_b128_T53', 'dilated', 53, 0.25, True),
    ('dense_333_128ch_b128_T27', 'dense', 27, 0.25, True),
    ('o1f_27f_128ch_b128_graphed', 'o1f', 27, 0.05, True),
    ('o1f_27f_128ch_b128_eager', 'o1f', 27, 0.05, False),
]


def worker(steps):
    import torch
    sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
    sys.path.insert(0, REPO)
    from gast_b200 import synth
    from gast_b200.trainer import DataParallelTrainer, GraphedTrainer
    from gast_b200.pipeline import FusedAdam
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    J, B = 17, 128
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))

    def make(kind, fw, ch, drop):
        if kind == 'o1f':
            m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, dropout=drop, channels=ch)
        else:
            m = SpatioTemporalModel(adj, J, 2, J, fw, dropout=drop, channels=ch, dense=(kind == 'dense'))
        synth.randomize_module(m, 1)
        return m.cuda()

    out = {'lib': os.environ.get('GAST_B200_LIB', 'in-tree')}
    for name, kind, T, drop, graphed in CASES:
        m = make(kind, [3, 3, 3], 128, drop)
        T_out = T - 26 if kind != 'o1f' else 1
        x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=3)).cuda()
        y = torch.randn(B, T_out, J, 3, generator=torch.Generator().manual_seed(4)).cuda()
        opt = lambda ps: FusedAdam(ps, lr=1e-3, amsgrad=True)  # noqa: E731
        tr = GraphedTrainer(m, opt, (B, T, J, 2), (B, T_out, J, 3)) if graphed else DataParallelTrainer(m, opt)
        for _ in range(3):
            tr.step(x, y)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            tr.step(x, y)
        e1.record()
        torch.cuda.synchronize()
        out[name] = round(e0.elapsed_time(e1) / steps, 4)
        del tr, m
        torch.cuda.empty_cache()
    # workspace queries: DESIGN.md §11 (Optimized1f 27f/128ch) and §11.1 (dilated 27f/128ch and 81f/64ch)
    ws = {}
    m = make('o1f', [3, 3, 3], 128, 0.05).eval()
    with torch.no_grad():
        m(torch.from_numpy(synth.synth_input(1, 27, J, 2, seed=1)).cuda())
    h = list(m.__dict__['_gast_handles'].values())[0]
    ws['o1f_128ch_train_b128'] = int(h.lib.gast_train_workspace_bytes(h.h, 128, 27, 0.05))
    for b in (128, 4096):
        ws['o1f_128ch_eval_backward_b%d' % b] = int(h.lib.gast_eval_backward_workspace_bytes(h.h, b, 27, 1))
    for fw, ch in (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
        m = make('dilated', fw, ch, 0.25).eval()
        rf = m.receptive_field()
        with torch.no_grad():
            m(torch.from_numpy(synth.synth_input(1, rf, J, 2, seed=1)).cuda())
        h = list(m.__dict__['_gast_handles'].values())[0]
        tag = '%df_%dch' % (rf, ch)
        ws[tag + '_train_b128_T%d' % rf] = int(h.lib.gast_train_workspace_bytes(h.h, 128, rf, 0.25))
        for T in (rf + 1000, rf + 2000):
            ws[tag + '_eval_backward_T%d' % T] = int(h.lib.gast_eval_backward_workspace_bytes(h.h, 1, T, 0))
        for mf in (256, 1024, 2048):
            ws[tag + '_chunked_mf%d' % mf] = int(h.lib.gast_chunked_workspace_bytes(h.h, 1, 10 ** 6, 0, mf, 1))
    out['workspace_bytes'] = ws
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', default=[], help='LABEL=PATH of a libgast_b200.so (repeat)')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--out', default=None)
    ap.add_argument('--worker', action='store_true', help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        return worker(a.steps)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('repeatable_grad_bench: needs a CUDA device')
    sys.path.insert(0, os.path.join(REPO, 'tools'))
    from chunk_stream_bench import card
    libs = [s.split('=', 1) for s in a.lib] or [['in-tree', '']]
    out = open(a.out, 'w') if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + '\n')
            out.flush()

    emit({'card': card()})
    res = {label: [] for label, _ in libs}
    for r in range(a.rounds):
        for label, path in libs:
            env = dict(os.environ)
            if path:
                env['GAST_B200_LIB'] = os.path.abspath(path)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', '--steps', str(a.steps)],
                               env=env, capture_output=True, text=True)
            if p.returncode != 0:
                raise SystemExit('worker %s failed:\n%s' % (label, p.stderr[-4000:]))
            d = json.loads(p.stdout.strip().splitlines()[-1])
            d.update({'build': label, 'round': r})
            emit(d)
            res[label].append(d)
    for name, *_ in CASES:
        for label, _ in libs:
            ms = [d[name] for d in res[label]]
            emit({'case': name, 'build': label, 'ms_per_step_median': statistics.median(ms),
                  'ms_per_step_range': [min(ms), max(ms)]})
    emit({'card': card()})


if __name__ == '__main__':
    main()
