"""GPU: scoring a synthetic Human3.6M-sized test set, the reference's way against evaluate_sequences.

The test set: `--seqs` sequences of 1000-5000 frames (seeded), 17 joints, 15 groups ("actions"), lifted by the
27-frame/128ch SpatioTemporalModel with synthetic weights, with and without test-time augmentation.  Two ways to
score it, alternated `--reps` times in one process:
  * reference: the staged, unchanged main.evaluate (oracle/_ref/main.py) over an UnchunkedGenerator per group, as
    trainval.py's run_evaluation calls it: one whole-sequence forward per sequence over the drop-in model, one
    `.item()` per sequence, p_mpjpe as the reference's float32 numpy SVD on the host;
  * device: gast_b200.evaluation.evaluate_sequences (lift_sequences + one gast_pose_metrics call).
Prints one JSON line per run with both action-wise e1 / e2 (mm) and both wall times (host clock around work that ends
in a device synchronise), the first line with the card's name and power limit read in the same run, and one line
with the time of the scoring call alone (CUDA events, mean of 5 after a warm-up).  Needs
oracle/_ref/ (build() stages it); without it only the device path runs.

    python tools/eval_bench.py [--seqs 240] [--reps 3]
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
sys.path[:0] = [PKG, REPO]
from gast_b200 import synth  # noqa: E402
from gast_b200 import pipeline as P  # noqa: E402
from gast_b200.evaluation import AUC_THRESHOLDS, evaluate_sequences  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModel  # noqa: E402

KL, KR = [4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]


def card():
    d = {'name': torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.sm',
                            '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30)
        d['power_limit_w'], d['sm_mhz'] = [v.strip() for v in r.stdout.strip().split(',')]
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return d


def test_set(n, seed=0):
    rs = np.random.RandomState(seed)
    lengths = rs.randint(1000, 5001, n)
    p2 = [synth.synth_input(1, int(T), 17, 2, seed=seed + 1 + i)[0] for i, T in enumerate(lengths)]
    p3 = [(0.25 * rs.standard_normal((T, 17, 3)) + rs.uniform(-1, 1, (1, 1, 3))).astype(np.float32) for T in lengths]
    groups = ['action%02d' % (i % 15) for i in range(n)]
    return p2, p3, groups


def reference_main():
    if not os.path.exists(os.path.join(REF, 'main.py')):
        return None, None
    sys.path[:] = [PKG, REF] + [p for p in sys.path if p not in (PKG, REF)]
    import main                                        # oracle/_ref/main.py, unchanged
    from common.generators import UnchunkedGenerator   # oracle/_ref/common/generators.py
    return main, UnchunkedGenerator


def run_reference(main, Gen, m, p2, p3, groups, augment):
    pad = (m.receptive_field() - 1) // 2
    e1s, e2s = [], []
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        for g in dict.fromkeys(groups):
            idx = [i for i, x in enumerate(groups) if x == g]
            gen = Gen(None, [p3[i] for i in idx], [p2[i] for i in idx], pad=pad, causal_shift=0, augment=augment,
                      kps_left=KL, kps_right=KR, joints_left=KL, joints_right=KR)
            e1, e2 = main.evaluate(gen, m, KL, KR, g)
            e1s.append(e1)
            e2s.append(e2)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, float(np.mean(e1s)), float(np.mean(e2s))


def run_device(m, p2, p3, groups, augment):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = evaluate_sequences(m, p2, p3, groups, augment=augment, kps_left=KL, kps_right=KR, joints_left=KL,
                             joints_right=KR)
    torch.cuda.synchronize()
    e1, e2 = res.action_wise()
    return time.perf_counter() - t0, e1 * 1000, e2 * 1000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--seqs', type=int, default=240, help='sequences in the test set')
    ap.add_argument('--reps', type=int, default=3, help='alternated runs of each path')
    args = ap.parse_args()
    print(json.dumps({'card': card()}), flush=True)
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), [], []))
    m = SpatioTemporalModel(adj, 17, 2, 17, [3, 3, 3], channels=128)
    synth.randomize_module(m, 3)
    m = m.cuda().eval()
    p2, p3, groups = test_set(args.seqs)
    print(json.dumps({'sequences': len(p2), 'frames': int(sum(len(p) for p in p2)), 'groups': len(set(groups))}),
          flush=True)
    # the scoring alone: one gast_pose_metrics call over every frame (P-MPJPE and the 31 AUC thresholds on)
    tgt = torch.as_tensor(np.concatenate(p3)).cuda()
    pred = tgt + 0.05 * torch.randn(tgt.shape, generator=torch.Generator().manual_seed(1)).cuda()
    seg = np.concatenate([[0], np.cumsum([len(p) for p in p3])])
    score = lambda: P.pose_metrics(pred, tgt, seg, AUC_THRESHOLDS, zero_root=True)  # noqa: E731
    score()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        score()
    e1.record()
    torch.cuda.synchronize()
    print(json.dumps({'pose_metrics_ms': e0.elapsed_time(e1) / 5, 'frames': int(tgt.shape[0])}), flush=True)
    del tgt, pred
    ref_main, Gen = reference_main()
    for augment in (False, True):
        short = [x[:300] for x in p2[:4]], [x[:300] for x in p3[:4]], groups[:4]      # warm-up: modules, allocator
        run_device(m, *short, augment)
        if ref_main is not None:
            run_reference(ref_main, Gen, m, *short, augment)
        for rep in range(args.reps):
            out = {'augment': augment, 'rep': rep}
            out['device_s'], out['device_e1'], out['device_e2'] = run_device(m, p2, p3, groups, augment)
            if ref_main is not None:
                out['reference_s'], out['reference_e1'], out['reference_e2'] = run_reference(ref_main, Gen, m, p2, p3,
                                                                                            groups, augment)
                out['speedup'] = out['reference_s'] / out['device_s']
            print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
