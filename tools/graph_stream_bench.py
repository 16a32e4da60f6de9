"""GPU: a real-time tick replayed from a CUDA graph (GraphedPoseStream) against the eager tick (PoseStream.push, plus
PoseStream.peek when the tick peeks), K = 1 frame per stream, every stream pushing.  27-frame/128ch and 81-frame/64ch
non-causal models; n = 1, 4, 16, 64, 256, 1024 streams; augment off and on; no peek and a peek of `latency` frames.
For each configuration the two paths alternate in one process, three windows each, and each window reports
  * wall_ms: host clock per tick over a window of ticks closed by a device synchronise (what a caller's loop sees);
  * device_ms: CUDA events per tick, around each replay for the graph and around each eager call (push + peek) for
    the eager path.  An eager call enqueues its kernels more slowly than the GPU runs them, so its event span also
    holds the gaps between its kernels: it is the call's time on the stream, not its kernels' busy time;
  * launches per tick.
Prints one JSON line per configuration (medians of the three windows, and every window), the first line with the
card's name, power limit and SM clock read in the same run.

    python tools/graph_stream_bench.py [--quick] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
from chunk_stream_bench import card  # noqa: E402
from gast_b200 import synth  # noqa: E402
from gast_b200.realtime import GraphedPoseStream, PoseStream  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f  # noqa: E402

WINDOWS = 3


def window(tick, spans, ticks):
    """-> (wall ms per tick, device ms per tick): `ticks` calls of tick(), closed by a synchronise; spans() -> the
    event pairs recorded by those calls"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(ticks):
        tick()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / ticks
    return wall, sum(a.elapsed_time(b) for a, b in spans()) / ticks


def measure(m, n, augment, peek, ticks):
    J = 17
    x1 = torch.from_numpy(synth.synth_input(n, 1, J, 2, seed=10)).cuda()           # (n, 1, J, 2)
    lat = (m.receptive_field() - 1) // 2
    P = lat if peek else 0
    eager = PoseStream(m, n, augment=augment)
    graph = GraphedPoseStream(m, n, augment=augment, K=1, peek=P)
    ev = {'eager': [], 'graph': []}

    def pair(key):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev[key].append((a, b))
        return a, b

    def eager_tick():
        a, b = pair('eager')
        a.record()
        eager.push(x1[:, 0])
        launches = eager.last_launches
        if P:
            eager.peek(P)
            launches += eager.last_launches
        b.record()
        eager_tick.launches = launches

    def graph_tick():
        graph.push(x1)

    graph.push(x1)                                      # the capture
    replay = graph.graph.replay

    def timed_replay():                                 # events around the replay only
        a, b = pair('graph')
        a.record()
        replay()
        b.record()
    graph.graph.replay = timed_replay
    for _ in range(5):
        eager_tick()
        graph_tick()
    res = {'eager': [], 'graph': []}
    for _ in range(WINDOWS):
        for key, fn in (('eager', eager_tick), ('graph', graph_tick)):
            ev[key] = []
            res[key].append(window(fn, lambda: ev[key], ticks))
    med = lambda v: sorted(v)[len(v) // 2]   # noqa: E731
    out = {'streams': n, 'augment': augment, 'peek': P}
    for key, launches in (('eager', eager_tick.launches), ('graph', graph.last_launches)):
        out[key] = {'wall_ms': med([w for w, _ in res[key]]), 'device_ms': med([d for _, d in res[key]]),
                    'launches': launches, 'windows': res[key]}
    out['wall_speedup'] = out['eager']['wall_ms'] / out['graph']['wall_ms']
    del eager, graph
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--quick', action='store_true', help='the 27-frame model, n <= 64, no augment')
    ap.add_argument('--out', help='also append the JSON lines to this file')
    args = ap.parse_args()
    sink = open(args.out, 'a') if args.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if sink:
            sink.write(line + '\n')
            sink.flush()
    emit({'card': card()})
    J = 17
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    models = (([3, 3, 3], 128),) if args.quick else (([3, 3, 3], 128), ([3, 3, 3, 3], 64))
    for fw, ch in models:
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=False, channels=ch, dropout=0.25)
        synth.randomize_module(m, 2)
        m = m.cuda().eval()
        name = '%d-frame/%dch non-causal' % (m.receptive_field(), ch)
        with torch.no_grad():
            for augment in ((False,) if args.quick else (False, True)):
                for peek in (False, True):
                    for n in ((1, 4, 16, 64) if args.quick else (1, 4, 16, 64, 256, 1024)):
                        rec = measure(m, n, augment, peek, 100 if n <= 64 else 30)
                        rec['model'] = name
                        emit(rec)


if __name__ == '__main__':
    main()
