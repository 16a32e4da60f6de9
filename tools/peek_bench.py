"""GPU: what a provisional pose costs a live caller.  ms per `PoseStream.push` and per `push` followed by `peek(K)`
(gast_stream_peek_subset on its lockstep branch: the kernels of gast_stream_peek) for the 27-frame/128ch and
81-frame/64ch non-causal models, n = 1, 64, 1024 streams, K = 1, latency/2 and latency, with and without
augmentation.  Prints one JSON line per measurement, the first with the card's
name, power limit and SM clock read in the same run.  CUDA events after a warm-up; each stream has pushed more than
`latency` frames, so that every peek has poses due.

    python tools/peek_bench.py [--quick]
"""
import argparse
import json
import os
import sys

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--quick', action='store_true', help='n <= 64 only')
    args = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    J = 17
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    for fw, ch in (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=False, channels=ch, dropout=0.25)
        synth.randomize_module(m, 2)
        m = m.cuda().eval()
        name = '%d-frame/%dch non-causal' % (m.receptive_field(), ch)
        for augment in (False, True):
            for n in ((1, 64) if args.quick else (1, 64, 1024)):
                ps = PoseStream(m, n, augment=augment)
                lat = ps.latency
                warm = torch.from_numpy(synth.synth_input(n, 2 * lat, J, 2, seed=10)).cuda()
                ps.push_frames(warm)                         # every stream live with more than `latency` frames
                x = warm[:, -1]
                calls = 20 if n >= 1024 else 100
                push_ms = timed(lambda: ps.push(x), 10, calls)
                rec = {'model': name, 'augment': augment, 'streams': n, 'push_ms': push_ms,
                       'push_launches': ps.last_launches}
                for K in sorted({1, lat // 2, lat}):
                    def both():
                        ps.push(x)
                        ps.peek(K)
                    ms = timed(both, 5, calls)
                    rec['K=%d' % K] = {'push_peek_ms': ms, 'peek_ms': ms - push_ms, 'peek_launches': ps.last_launches}
                print(json.dumps(rec), flush=True)
                del ps
                torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
