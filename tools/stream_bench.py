"""GPU: frames/s of the real-time path (SURVEY.md 8f N4) -- O(1)-per-frame rings (CausalStream, gast_stream_push)
against recomputing the receptive field for every frame (WindowStream: what the reference's real-time loop does,
gen_skes.py:43-69), for 1 and many concurrent streams, 27-frame/128ch and 81-frame/64ch causal models; then the
delayed stream of the non-causal models of the same sizes (PoseStream, gast_stream_push_ex), with and without
test-time augmentation."""
import json
import os
import sys
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
from gast_b200 import synth  # noqa: E402
from gast_b200.realtime import CausalStream, PoseStream, WindowStream  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f  # noqa: E402


def run(stream, frames, warm, reps):
    for t in range(warm):
        stream.push(frames[t % len(frames)])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for t in range(reps):
        stream.push(frames[t % len(frames)])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    J = 17
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    out = []
    for fw, ch in (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=True, channels=ch, dropout=0.25)
        synth.randomize_module(m, 2)
        m = m.cuda().eval()
        for n in (1, 64, 1024):
            frames = [torch.from_numpy(synth.synth_input(n, 1, J, 2, seed=10 + i)[:, 0]).cuda() for i in range(8)]
            ms_o1 = run(CausalStream(m, n), frames, 100, 200 if n < 1024 else 50)
            ms_win = run(WindowStream(m, n), frames, 20, 50 if n < 1024 else 10)
            rec = {'model': '%d-frame/%dch causal' % (m.receptive_field(), ch), 'streams': n,
                   'o1_ms_per_frame': ms_o1, 'o1_frames_per_s': n / ms_o1 * 1e3,
                   'window_ms_per_frame': ms_win, 'window_frames_per_s': n / ms_win * 1e3, 'speedup': ms_win / ms_o1}
            print(json.dumps(rec), flush=True)
            out.append(rec)
    for fw, ch in (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
        m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=False, channels=ch, dropout=0.25)
        synth.randomize_module(m, 2)
        m = m.cuda().eval()
        for augment in (False, True):
            for n in (1, 64, 1024):
                frames = [torch.from_numpy(synth.synth_input(n, 1, J, 2, seed=10 + i)[:, 0]).cuda() for i in range(8)]
                ms = run(PoseStream(m, n, augment=augment), frames, 100, 200 if n < 1024 else 50)
                rec = {'model': '%d-frame/%dch non-causal' % (m.receptive_field(), ch), 'augment': augment,
                       'streams': n, 'pose_ms_per_frame': ms, 'pose_frames_per_s': n / ms * 1e3}
                print(json.dumps(rec), flush=True)
                out.append(rec)


if __name__ == '__main__':
    main()
