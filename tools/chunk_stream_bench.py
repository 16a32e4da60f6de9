"""GPU: K frames per stream in one call (PoseStream.push_frames, the kernels of gast_stream_push_chunk) against one
push per frame (K = 1 is `push`), and bounded-memory whole-sequence lifting (lift_sequences) against the
whole-sequence forward (tta.evaluate_sequence): time, peak device memory and the largest difference of their poses.
Prints one JSON line per measurement, the first with the card's name and power limit read in the same run.  CUDA
events after a warm-up.

    python tools/chunk_stream_bench.py [--quick] [--frames 20000]
"""
import argparse
import json
import os
import subprocess
import sys
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
from gast_b200 import synth, tta  # noqa: E402
from gast_b200.realtime import PoseStream, SYMMETRY, lift_sequences  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f  # noqa: E402


def card():
    d = {'name': torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.sm',
                            '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30)
        d['power_limit_w'], d['sm_mhz'] = [v.strip() for v in r.stdout.strip().split(',')]
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return d


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
    ap.add_argument('--quick', action='store_true', help='fewer configurations (n <= 64)')
    ap.add_argument('--frames', type=int, default=20000, help='length of the lifted sequence')
    ap.add_argument('--lift-only', action='store_true', help='only the whole-sequence comparison')
    args = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    J = 17
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    for fw, ch in () if args.lift_only else (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=False, channels=ch, dropout=0.25)
        synth.randomize_module(m, 2)
        m = m.cuda().eval()
        name = '%d-frame/%dch non-causal' % (m.receptive_field(), ch)
        for augment in (False, True):
            for n in ((1, 64) if args.quick else (1, 64, 1024)):
                for K in (1, 8, 64, 256):
                    if n * K > 64 * 1024:        # keep the workspace within a few GB
                        continue
                    x = torch.from_numpy(synth.synth_input(n, K, J, 2, seed=10)).cuda()
                    ps = PoseStream(m, n, augment=augment)
                    calls = max(3, min(200, 4096 // K))
                    ms = timed(lambda: ps.push_frames(x), max(3, calls // 4), calls)
                    rec = {'model': name, 'augment': augment, 'streams': n, 'K': K, 'ms_per_call': ms,
                           'frames_per_s': n * K / ms * 1e3, 'launches': ps.last_launches}
                    print(json.dumps(rec), flush=True)
                    del ps
                    torch.cuda.empty_cache()
    # one long sequence: lift_sequences (bounded scratch) against the whole-sequence forward
    kl, kr = SYMMETRY[17]
    for fw, ch in (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
        m = SpatioTemporalModel(adj, J, 2, J, fw, causal=False, channels=ch, dropout=0.25)
        synth.randomize_module(m, 2)
        m = m.cuda().eval()
        seq = synth.synth_input(1, args.frames, J, 2, seed=3)[0]
        rec = {'model': '%d-frame/%dch non-causal, TTA' % (m.receptive_field(), ch), 'frames': args.frames}
        res = {}
        for what, fn in (('whole', lambda: tta.evaluate_sequence(m, seq, kl, kr, kl, kr)),
                         ('lift', lambda: lift_sequences(m, [seq], n_streams=1, chunk=1024, augment=True)[0])):
            for rep in range(2):                   # the first call includes workspaces the handle keeps
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                y = fn()
                e1.record()
                torch.cuda.synchronize()
                sfx = '_first' if rep == 0 else ''
                rec[what + sfx + '_ms'] = e0.elapsed_time(e1)
                rec[what + sfx + '_peak_mb'] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
                res[what] = y
        d = (res['lift'] - res['whole']).abs().max().item()
        rec['max_abs_diff'] = d
        rec['max_rel_diff'] = d / res['whole'].abs().max().item()
        print(json.dumps(rec), flush=True)
        del res
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
