"""GPU: what a tick costs when only some streams have a frame.  On a 1024-stream state, ms per `PoseStream.push` of
m = 1, 16, 64, 256, 1024 listed streams at their own frame counts (gast_stream_push_subset, K = 1), against the two
baselines a caller had before: the lockstep `push` of all 1024 streams (held streams included) and a `push` on a state
of m streams only (the floor).  27-frame/128ch and 81-frame/64ch non-causal models, with and without augmentation.
Prints one JSON line per measurement, the first with the card's name, power limit and SM clock read in the same run.
CUDA events after a warm-up.

    python tools/subset_stream_bench.py [--quick]
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
from chunk_stream_bench import card, timed  # noqa: E402
from gast_b200 import synth  # noqa: E402
from gast_b200.realtime import PoseStream  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f  # noqa: E402

N = 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--quick', action='store_true', help='the 27-frame model without augmentation only')
    args = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    J = 17
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    rng = np.random.default_rng(0)
    models = (([3, 3, 3], 128),) if args.quick else (([3, 3, 3], 128), ([3, 3, 3, 3], 64))
    for fw, ch in models:
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=False, channels=ch, dropout=0.25)
        synth.randomize_module(m, 2)
        m = m.cuda().eval()
        name = '%d-frame/%dch non-causal' % (m.receptive_field(), ch)
        for augment in ((False,) if args.quick else (False, True)):
            x = torch.from_numpy(synth.synth_input(N, 1, J, 2, seed=10)[:, 0].copy()).cuda()
            ps = PoseStream(m, N, augment=augment)
            lock_ms = timed(lambda: ps.push(x), 5, 20)
            print(json.dumps({'model': name, 'augment': augment, 'what': 'lockstep push', 'streams': N,
                              'ms_per_call': lock_ms, 'frames_per_s': N / lock_ms * 1e3,
                              'launches': ps.last_launches}), flush=True)
            for mm in (1, 16, 64, 256, N):
                sel = sorted(rng.choice(N, size=mm, replace=False).tolist())
                xs = x[:mm].contiguous()
                ps.push(xs, streams=sel)                           # the counts differ from here on
                calls = 20 if mm >= 256 else 100
                sub_ms = timed(lambda: ps.push(xs, streams=sel), 5, calls)
                rec = {'model': name, 'augment': augment, 'what': 'subset push', 'streams': N, 'm': mm,
                       'ms_per_call': sub_ms, 'frames_per_s': mm / sub_ms * 1e3, 'launches': ps.last_launches}
                floor = PoseStream(m, mm, augment=augment)
                rec['floor_push_ms'] = timed(lambda: floor.push(xs), 5, calls)
                rec['lockstep_push_ms'] = lock_ms
                print(json.dumps(rec), flush=True)
                del floor
                torch.cuda.empty_cache()
            del ps
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
