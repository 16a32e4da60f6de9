"""Eval-mode gradients in bounded memory (engine.run_model_chunked, gast_eval_backward_chunked) against the unchunked
call (model(x) with autograd, gast_eval_backward), on the dilated SpatioTemporalModel, 27-frame/128ch and
81-frame/64ch:
  * where both fit, alternated in one process: a forward + backward of one recording and of a batch of
    receptive-field clips, ms per output frame (host clock around the call, closed by a synchronise; median of the
    rounds) and the peak of torch.cuda.max_memory_allocated over the call;
  * a long recording chunked only, and the per-frame workspace of the unchunked call from its sizing query
    (gast_eval_backward_workspace_bytes), with the length at which that query passes the device's memory.
Prints one JSON line per measurement, the first with the card's name, power limit and SM clock read in the same run.

    python tools/chunked_grad_bench.py [--rounds N] [--long T] [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
from chunk_stream_bench import card  # noqa: E402
from gast_b200 import engine, synth  # noqa: E402


def model(fw, ch):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    m = SpatioTemporalModel(adj, 17, 2, 17, fw, channels=ch)
    synth.randomize_module(m, 5)
    return m.cuda().eval()


def call(m, x, dy, max_frames):
    """forward + backward of (y * dy).sum() through model(x) (max_frames None) or run_model_chunked"""
    m.zero_grad(set_to_none=True)
    xx = x.detach().requires_grad_()
    y = m(xx) if max_frames is None else engine.run_model_chunked(m, xx, max_frames)
    y.backward(dy)


def measure(m, x, dy, max_frames):
    """(seconds, peak bytes above what was allocated before) of one call"""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    call(m, x, dy, max_frames)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated() - base


def compare(m, name, B, T, variants, rounds, emit):
    """variants: [(distinct label, max_frames or None)], alternated round by round"""
    x = torch.from_numpy(synth.synth_input(B, T, 17, 2, seed=1)).cuda()
    with torch.no_grad():
        T_out = m(x).shape[1]
    dy = torch.randn(B, T_out, 17, 3, generator=torch.Generator().manual_seed(2)).cuda()
    for _, mf in variants:                            # warm every shape
        call(m, x, dy, mf)
    res = {label: [] for label, _ in variants}
    peak = {}
    for _ in range(rounds):
        for label, mf in variants:
            s, p = measure(m, x, dy, mf)
            res[label].append(s)
            peak[label] = max(peak.get(label, 0), p)
    for label, mf in variants:
        ms = [1e3 * s / (B * T_out) for s in res[label]]
        emit({'model': name, 'B': B, 'T': T, 'T_out': T_out, 'call': label, 'max_frames': mf,
              'ms_per_output_frame_median': round(statistics.median(ms), 5),
              'ms_per_output_frame_range': [round(min(ms), 5), round(max(ms), 5)],
              'ms_per_call_median': round(1e3 * statistics.median(res[label]), 3),
              'peak_mib': round(peak[label] / 2 ** 20, 1)})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--long', type=int, default=100000, help='frames of the chunked-only recording')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('chunked_grad_bench: needs a CUDA device')
    out = open(a.out, 'w') if a.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if out:
            out.write(line + '\n')
            out.flush()

    emit({'card': card()})
    total = torch.cuda.get_device_properties(0).total_memory
    for fw, ch in (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
        m = model(fw, ch)
        rf = m.receptive_field()
        name = '%d-frame/%dch dilated' % (rf, ch)
        x1 = torch.from_numpy(synth.synth_input(1, rf, 17, 2, seed=1)).cuda()
        with torch.no_grad():
            m(x1)
        h = list(m.__dict__['_gast_handles'].values())[0]
        q = lambda T: int(h.lib.gast_eval_backward_workspace_bytes(h.h, 1, T, 0))
        per_frame = (q(rf + 2000) - q(rf + 1000)) / 1000.0
        emit({'model': name, 'unchunked_eval_backward_workspace_bytes_per_frame': round(per_frame),
              'unchunked_query_passes_device_memory_at_frames': int((total - q(rf)) / per_frame) + rf,
              'device_memory_bytes': total,
              'chunked_workspace_bytes': {mf: int(h.lib.gast_chunked_workspace_bytes(h.h, 1, 10 ** 6, 0, mf, 1))
                                          for mf in (256, 1024, 2048)}})
        # one recording, and a batch of receptive-field clips (one output each, the strided schedule)
        compare(m, name, 1, 4096 + rf - 1, [('unchunked', None), ('chunked 1024', 1024), ('chunked 2048', 2048)],
                a.rounds, emit)
        compare(m, name, 1024, rf, [('unchunked', None), ('chunked 256', 256)], a.rounds, emit)
        # a long recording, chunked only
        T = a.long + rf - 1
        x = torch.from_numpy(synth.synth_input(1, T, 17, 2, seed=3)).cuda()
        dy = torch.randn(1, a.long, 17, 3, generator=torch.Generator().manual_seed(4)).cuda()
        call(m, x, dy, 2048)
        s, p = measure(m, x, dy, 2048)
        emit({'model': name, 'B': 1, 'T': T, 'T_out': a.long, 'call': 'chunked', 'max_frames': 2048,
              'ms_per_output_frame': round(1e3 * s / a.long, 5), 'ms_per_call': round(1e3 * s, 1),
              'peak_mib': round(p / 2 ** 20, 1), 'unchunked_query_gib': round(q(T) / 2 ** 30, 1)})
        del m, x, dy
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
