"""GPU: one training epoch and one validation pass of trainval.py's loop, three ways, on a synthetic training split.

The split: `--seqs` sequences of `--frames` frames (seeded), 17 joints, flip augmentation (both halves of every
chunk, as trainval's --data-augmentation does), lifted by Optimized1f 27f/128ch (dropout 0) at batch `--batch`.
Alternated `--reps` times in one process, each way keeping its own model, optimiser and generator from the same
start, so that rep r is epoch r + 1 of each:
  (a) the staged, unchanged main.train (oracle/_ref/main.py) with the reference's host ChunkedGenerator and
      torch.optim.Adam(amsgrad=True): what trainval.py runs over the drop-in today;
  (b) main.train with the device ChunkedGenerator and FusedAdam (tests/epochref.py: main.train's own code with its
      host-array conversions as identities, the edit INTEGRATION.md §3 describes);
  (c) gast_b200.training.EpochTrainer.train_epoch.
(b) and (c) must return the same epoch loss bit for bit; the lr decays by 0.95 between epochs as trainval's does.
Then main.eval (reference UnchunkedGenerators over a test split of the same size and the training split) against
EpochTrainer.eval_epoch.  Wall times are host clocks around work that ends in a device synchronise.  Prints JSON
lines: the card's name, power limit and SM clock read in the same run first, then one line per rep.

    python tools/epoch_bench.py [--seqs 64] [--frames 2000] [--batch 128] [--reps 3]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, 'gast-net-3dposeestimation_b200')
REF = os.path.join(REPO, 'oracle', '_ref')
sys.path[:0] = [PKG, REPO, os.path.join(REPO, 'tests')]
from gast_b200 import synth, training  # noqa: E402
from gast_b200 import pipeline as P  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f  # noqa: E402
from device.common.generators import ChunkedGenerator as DeviceChunked  # noqa: E402
import epochref  # noqa: E402

KL, KR = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]
DECAY = 0.95


def card():
    d = {'name': torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30)
        d['power_limit_w'], d['sm_mhz'], d['sm_max_mhz'] = [v.strip() for v in r.stdout.strip().split(',')]
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return d


def split(n, T, seed):
    rs = np.random.RandomState(seed)
    p2 = [synth.synth_input(1, T, 17, 2, seed=seed + 1 + i)[0] for i in range(n)]
    p3 = [(0.25 * rs.standard_normal((T, 17, 3)) + rs.uniform(-1, 1, (1, 1, 3))).astype(np.float32) for _ in range(n)]
    return p2, p3


def models():
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), KL, KR))
    m = SpatioTemporalModelOptimized1f(adj, 17, 2, 17, [3, 3, 3], dropout=0.0, channels=128)
    synth.randomize_module(m, 3)
    mp = SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], dropout=0.0, channels=128)
    return m.cuda().train(), mp.cuda()


def gen_kw():
    return dict(pad=13, causal_shift=0, shuffle=True, random_seed=1234, augment=True, kps_left=KL, kps_right=KR,
                joints_left=KL, joints_right=KR)


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seqs', type=int, default=64)
    ap.add_argument('--frames', type=int, default=2000)
    ap.add_argument('--batch', type=int, default=128)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not os.path.exists(os.path.join(REF, 'main.py')):
        sys.exit('epoch_bench: oracle/_ref/ is not staged (python __graft_entry__.py build with an original checkout)')
    print(json.dumps({'card': card()}), flush=True)
    sys.path[:] = [PKG, REF] + [p for p in sys.path if p not in (PKG, REF)]
    import main as ref_main                                  # oracle/_ref/main.py, unchanged
    from common.generators import ChunkedGenerator as HostChunked, UnchunkedGenerator
    p2, p3 = split(args.seqs, args.frames, 0)
    t2, t3 = split(args.seqs, args.frames, 10_000)
    (ma, mpa), (mb, _), (mc, mpc) = models(), models(), models()
    ga = HostChunked(args.batch, None, p3, p2, 1, **gen_kw())
    gb = DeviceChunked(args.batch, None, p3, p2, 1, **gen_kw())
    gc = DeviceChunked(args.batch, None, p3, p2, 1, **gen_kw())
    oa = torch.optim.Adam(ma.parameters(), lr=1e-3, amsgrad=True)
    ob = P.FusedAdam(mb.parameters(), lr=1e-3, amsgrad=True)
    oc = P.FusedAdam(mc.parameters(), lr=1e-3, amsgrad=True)
    build_s, tr = timed(lambda: training.EpochTrainer(mc, gc, oc))
    print(json.dumps({'sequences': args.seqs, 'frames_per_sequence': args.frames, 'batch': args.batch,
                      'pairs': len(gc.pairs), 'batches_per_epoch': gc.num_batches, 'trainer_build_s': build_s}),
          flush=True)
    for rep in range(args.reps):
        out = {'rep': rep}
        out['a_s'], out['a_loss'] = timed(lambda: ref_main.train(ma, ga, oa))
        out['b_s'], out['b_loss'] = timed(lambda: epochref.main_train_device(ref_main, mb, gb, ob))
        out['c_s'], out['c_loss'] = timed(tr.train_epoch)
        out['b_equals_c'] = out['b_loss'] == out['c_loss']
        out['a_over_c'], out['b_over_c'] = out['a_s'] / out['c_s'], out['b_s'] / out['c_s']
        out['c_ms_per_batch'] = 1000 * out['c_s'] / gc.num_batches
        for o in (oa, ob, oc):
            for g in o.param_groups:
                g['lr'] *= DECAY
        print(json.dumps(out), flush=True)
    for rep in range(args.reps):
        out = {'eval_rep': rep}
        tg = UnchunkedGenerator(None, t3, t2, pad=13, causal_shift=0, augment=False, kps_left=KL, kps_right=KR,
                                joints_left=KL, joints_right=KR)
        eg = UnchunkedGenerator(None, p3, p2, pad=13, causal_shift=0, augment=False)
        out['main_eval_s'], out['main_eval'] = timed(lambda: ref_main.eval(mc.state_dict(), mpa, tg, eg))
        out['eval_epoch_s'], out['eval_epoch'] = timed(lambda: tr.eval_epoch(mpc, t2, t3, p2, p3))
        out['speedup'] = out['main_eval_s'] / out['eval_epoch_s']
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
