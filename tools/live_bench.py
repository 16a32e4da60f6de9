"""Times the live tick (gast_b200.live.LiveTick) against the per-tick glue of existing calls it replaces.

For C cameras of 640 x 360 frames with num_person slots each, a causal 3-3-3 Optimized1f (32 channels, synthetic
weights) and light stand-in nets (tests/test_gpu_zz_live.py's: a Darknet that returns preset predictions, a pooled
HRNet), so that the pipeline's own cost is visible, the tool times per tick, host clock to a device synchronise:
  eager    LiveTick(graph=False);
  graphed  LiveTick(graph=True), one graph replay per tick;
  glue     letterbox -> person_boxes -> DeviceSort.update_chunk -> host_tracks -> host geometry -> crop_persons ->
           decode_heatmaps -> device.tools.preprocess -> PoseStream.push -> camera_to_world -> revise_skes_real_time
           (tests/test_gpu_zz_live.py's _Glue, which that test holds bit for bit to the tick).
The three are alternated in one process over --ticks ticks of walking persons, --rounds rounds, at C in {1, 4, 16}
and num_person in {1, 2}; the median per-tick time of each round is reported, with the library launches per tick
(the nets' own launches excluded).  The card's name and power limit are read in the same run.  Prints one JSON line.
Usage: python tools/live_bench.py [--rounds 3] [--ticks 60]
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
from gast_b200.live import LiveTick      # noqa: E402


def _card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                        '--format=csv,noheader'], text=True).strip().splitlines()[0]
    except Exception as e:                     # noqa: BLE001
        return 'unknown (%s)' % e


def _time(fn, frames, det, ticks):
    out = []
    for t, p in enumerate(ticks):
        det.preds.copy_(p)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn(frames)
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return float(np.median(out)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--ticks', type=int, default=60)
    a = ap.parse_args()
    card = _card()
    model = TL._model()
    rows = []
    for C in (1, 4, 16):
        frames, ticks = TL._scene(C, a.ticks, seed=C)
        for P in (1, 2):
            det, pose = TL._Darknet(C), TL._Pose().cuda()
            runs = {'eager': LiveTick(det, pose, model, C, (TL.W, TL.H), num_person=P),
                    'graphed': LiveTick(det, pose, model, C, (TL.W, TL.H), num_person=P, graph=True),
                    'glue': TL._Glue(det, pose, model, C, P, False)}
            for fn in runs.values():                       # warm-up: module loads, the capture
                for p in ticks[:3]:
                    det.preds.copy_(p)
                    fn(frames)
            ms = {k: [] for k in runs}
            for _ in range(a.rounds):
                for k, fn in runs.items():
                    ms[k].append(round(_time(fn, frames, det, ticks), 3))
            rows.append(dict(cameras=C, num_person=P, ms_per_tick=ms, launches=runs['eager'].last_launches))
            print('C=%d P=%d %s launches %d' % (C, P, ms, runs['eager'].last_launches), file=sys.stderr)
    print(json.dumps(dict(card=card, frame=[TL.W, TL.H], ticks=a.ticks, rows=rows)))


if __name__ == '__main__':
    main()
