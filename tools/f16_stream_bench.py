"""GPU: the fp16 inference precision (engine.set_precision(model, 'fp16')) against 'fp32' and 'tf32' on the real-time
paths and the headline forward of the 27-frame/128ch model, in one process: the card's name, power limit and SM clock,
then, with the three modes alternated three times each,
  * a lockstep single push of 1024 streams (PoseStream.push, gast_stream_push_ex);
  * push_frames of K = 256 frames into one stream (the chunk path);
  * a GraphedPoseStream tick of one stream with a 13-frame peek (K = 1);
  * the headline forward, 4096 clips x 27 frames x 17 joints;
and the stream state bytes per stream in each mode.  CUDA events after a warm-up; one JSON line per measurement.

    python tools/f16_stream_bench.py [--reps R]
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
from gast_b200 import engine, synth  # noqa: E402
from gast_b200.realtime import GraphedPoseStream, PoseStream  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModel  # noqa: E402
from launch_times import card  # noqa: E402

MODES = ('fp32', 'tf32', 'fp16')


def model():
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    m = SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], causal=False, dropout=0.05, channels=128)
    synth.randomize_module(m, 1)
    return m.cuda().eval()


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    args = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    m = model()
    n_lock, K_chunk, peek = 1024, 256, 13
    x_lock = torch.from_numpy(synth.synth_input(n_lock, 1, 17, 2, seed=1)[:, 0]).cuda()
    x_chunk = torch.from_numpy(synth.synth_input(1, K_chunk, 17, 2, seed=2)).cuda()
    x_tick = torch.from_numpy(synth.synth_input(1, 1, 17, 2, seed=3)).cuda()
    x_head = torch.from_numpy(synth.synth_input(4096, 27, 17, 2, seed=4)).cuda()
    pools = {}
    for mode in MODES:                     # a pool per mode: the fp16 pools keep their rings in fp16
        engine.set_precision(m, mode)
        pools[mode] = (PoseStream(m, n_lock), PoseStream(m, 1), GraphedPoseStream(m, 1, K=1, peek=peek))
        with torch.no_grad():
            for p in pools[mode][:2]:
                p.push_frames(x_chunk.expand(p.n, -1, -1, -1).contiguous()[:, :30])   # history in every ring slot
            pools[mode][2].push(x_tick)
        h = engine.model_handle(m, x_head.device)
        state = int(h.lib.gast_stream_state_bytes(h.h, 1))
        print(json.dumps({'mode': mode, 'stream_state_bytes_per_stream': state,
                          'state_bytes_1024': int(h.lib.gast_stream_state_bytes(h.h, 1024))}), flush=True)
    for rnd in range(3):
        for mode in MODES:
            engine.set_precision(m, mode)
            lock, one, graphed = pools[mode]
            with torch.no_grad():
                ms_lock = timed(lambda: lock.push(x_lock), 5, args.reps)
                ms_chunk = timed(lambda: one.push_frames(x_chunk), 2, max(5, args.reps // 5))
                ms_tick = timed(lambda: graphed.push(x_tick), 10, args.reps * 4)
                ms_head = timed(lambda: m(x_head), 3, max(5, args.reps // 5))
            print(json.dumps({'round': rnd, 'mode': mode,
                              'push_1024_ms': round(ms_lock, 4), 'push_1024_frames_per_s': round(n_lock / ms_lock * 1e3),
                              'push_frames_K256_ms': round(ms_chunk, 4),
                              'push_frames_K256_frames_per_s': round(K_chunk / ms_chunk * 1e3),
                              'graphed_tick_peek13_ms': round(ms_tick, 4),
                              'headline_ms': round(ms_head, 3), 'headline_clips_per_s': round(4096 / ms_head * 1e3)}),
                  flush=True)
    engine.set_precision(m, 'fp32')


if __name__ == '__main__':
    main()
