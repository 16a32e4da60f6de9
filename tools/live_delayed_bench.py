"""Times the delayed live tick of the non-causal models against the causal tick (gast_b200.live.LiveTick).

For C cameras of 640 x 360 frames with num_person slots each, 3-3-3 Optimized1f models (causal and non-causal,
synthetic weights, --channels each) and tests/test_gpu_zz_live.py's light stand-in nets, so that the pipeline's own
cost is visible, the tool times per tick, host clock to a device synchronise, eager and graphed:
  causal           the causal tick;
  delayed          the non-causal tick (latency 13), no provisional poses;
  delayed_now      the non-causal tick with lookahead 0 (a 13-frame provisional peek every tick).
The variants are alternated in one process over --ticks ticks of walking persons, --rounds rounds, at C x num_person
in {1 x 1, 4 x 2, 16 x 2}; the median per-tick time of each round is reported with the library launches per tick (the
nets' own excluded).  A separate torch.profiler run of graphed delayed_now ticks gives each kernel's share of the
tick's device time, and the share of the tail peek and of the provisional peek (the kernels of a
gast_stream_peek_device call and its TTA merge, found by launch order within the tick).  The card's name and power
limit are read in the same run.  Prints one JSON line; with --trace-dir, the profiler's Chrome traces are written
there.
Usage: python tools/live_delayed_bench.py [--rounds 3] [--ticks 40] [--channels 32 128] [--trace-dir DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))
import test_gpu_zz_live as TL            # noqa: E402
from common.graph_utils import adj_mx_from_skeleton   # noqa: E402
from common.skeleton import Skeleton     # noqa: E402
from gast_b200 import synth              # noqa: E402
from gast_b200.live import LiveTick      # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f   # noqa: E402


def _card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                        '--format=csv,noheader'], text=True).strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return 'unknown (%s)' % e


def _model(causal, channels):
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    m = SpatioTemporalModelOptimized1f(adj, 17, 2, 17, [3, 3, 3], causal=causal, channels=channels)
    synth.randomize_module(m, 3)
    return m.cuda().eval()


def _time(fn, frames, det, ticks):
    out = []
    for p in ticks:
        det.preds.copy_(p)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(frames)
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return float(np.median(out)) * 1e3


def _profile(model, C, P, frames, ticks, out_dir):
    """graphed delayed ticks with lookahead 0 under torch.profiler -> per-kernel device time shares"""
    from torch.profiler import ProfilerActivity, profile
    det, pose = TL._Darknet(C), TL._Pose().cuda()
    tick = LiveTick(det, pose, model, C, (TL.W, TL.H), num_person=P, graph=True, lookahead=0, delayed=True)
    for p in ticks[:3]:
        det.preds.copy_(p)
        tick(frames)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for p in ticks:
            det.preds.copy_(p)
            tick(frames)
        torch.cuda.synchronize()
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, 'live_delayed_trace_ch%d_C%d_P%d.json'
                                              % (int(model._gast_channels), C, P)))
    events = sorted((e for e in prof.events() if e.device_type.name == 'CUDA'), key=lambda e: e.time_range.start)
    per_tick = len(events) // len(ticks)
    total = sum(e.time_range.elapsed_us() for e in events)
    # the tick's kernels in launch order: gast_live_delayed_inputs, then the tail peek, the push and the provisional
    # peek (LiveTick.peek_launches kernels each)
    tail_n, push_n, now_n = tick.peek_launches
    groups = {'tail_peek': 0.0, 'push': 0.0, 'now_peek': 0.0}
    for j in [j for j, e in enumerate(events) if 'live_delayed_inputs' in e.name]:
        i = j + 1
        for name, cnt in (('tail_peek', tail_n), ('push', push_n), ('now_peek', now_n)):
            groups[name] += sum(e.time_range.elapsed_us() for e in events[i:i + cnt])
            i += cnt
    share = {}
    for e in events:
        share[e.name] = share.get(e.name, 0.0) + e.time_range.elapsed_us()
    top = sorted(share.items(), key=lambda kv: -kv[1])[:12]
    return dict(kernels_per_tick=per_tick, device_us_per_tick=round(total / len(ticks), 1),
                call_shares={k: round(v / total, 3) for k, v in groups.items()},
                top_shares=[(k[:80], round(v / total, 3)) for k, v in top])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--ticks', type=int, default=40)
    ap.add_argument('--channels', type=int, nargs='+', default=[32, 128])
    ap.add_argument('--trace-dir', default=None, help='write the profiler runs\' Chrome traces to this directory')
    a = ap.parse_args()
    card = _card()
    rows = []
    for ch in a.channels:
        causal, delayed = _model(True, ch), _model(False, ch)
        for C, P in ((1, 1), (4, 2), (16, 2)):
            frames, ticks = TL._scene(C, a.ticks, seed=C)
            det, pose = TL._Darknet(C), TL._Pose().cuda()
            runs = {}
            for g in (False, True):
                tag = 'graphed' if g else 'eager'
                kw = dict(num_person=P, graph=g)
                runs['causal_' + tag] = LiveTick(det, pose, causal, C, (TL.W, TL.H), **kw)
                runs['delayed_' + tag] = LiveTick(det, pose, delayed, C, (TL.W, TL.H), delayed=True, **kw)
                runs['delayed_now_' + tag] = LiveTick(det, pose, delayed, C, (TL.W, TL.H), lookahead=0,
                                                      delayed=True, **kw)
            for fn in runs.values():                       # warm-up: module loads, the capture
                for p in ticks[:3]:
                    det.preds.copy_(p)
                    fn(frames)
            ms = {k: [] for k in runs}
            for _ in range(a.rounds):
                for k, fn in runs.items():
                    ms[k].append(round(_time(fn, frames, det, ticks), 3))
            launches = {k: fn.last_launches for k, fn in runs.items() if k.endswith('eager')}
            rows.append(dict(channels=ch, cameras=C, num_person=P, ms_per_tick=ms, launches=launches))
            print('ch=%d C=%d P=%d %s %s' % (ch, C, P, ms, launches), file=sys.stderr)
    prof = {}
    for ch in a.channels:
        frames, ticks = TL._scene(16, 20, seed=16)
        prof['ch%d_16x2' % ch] = _profile(_model(False, ch), 16, 2, frames, ticks, a.trace_dir)
    print(json.dumps(dict(card=card, frame=[TL.W, TL.H], ticks=a.ticks, rows=rows, profile=prof)))


if __name__ == '__main__':
    main()
