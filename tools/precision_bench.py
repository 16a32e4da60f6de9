"""GPU: the single-pass TF32 precision (engine.set_precision(model, 'tf32')) and the half model (model.half(), fp16
weights, inputs and activations) against the default fp32-grade one, in one process: the card's name, power limit and
SM clock, then
  * the headline workload (4096 clips x 27 frames x 17 joints, 27-frame/128ch model) in fp32, TF32 and fp16,
    alternated three times each;
  * the 81-frame/64ch and 19-joint workloads;
  * per-GEMM device times of the headline forward in every mode (gast_set_timing);
  * PoseStream with 1024 streams (fp32 and TF32; half does not stream): single pushes and push_frames at K = 64;
  * the distance of the TF32 and fp16 poses from the fp32-grade ones: max |dy| / max |y| and the mean joint distance
    (the half model's input is the fp32 input rounded to fp16, its weights the fp32 model's rounded to fp16).
CUDA events after a warm-up; one JSON line per measurement.

    python tools/precision_bench.py [--headline-only] [--steps K]
"""
import argparse
import copy
import ctypes as C
import json
import os
import sys
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
from gast_b200 import engine, synth  # noqa: E402
from gast_b200.realtime import PoseStream  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModel  # noqa: E402
from launch_times import card, gemm_shapes  # noqa: E402


def model(J, fw, ch):
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    m = SpatioTemporalModel(adj, J, 2, J, fw, causal=False, dropout=0.05, channels=ch)
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


def clips_per_s(m, x, steps):
    with torch.no_grad():
        ms = timed(lambda: m(x), 3, steps)
    return x.shape[0] / ms * 1e3, ms


MODES = ('fp32', 'tf32', 'fp16')


def in_mode(m, mh, x, xh, mode):
    """(model, input) of a mode: the fp32 model at set_precision(mode), or its half copy mh with the fp16 input"""
    if mode == 'fp16':
        return mh, xh
    engine.set_precision(m, mode)
    return m, x


def emit(d):
    print(json.dumps(d), flush=True)


def accuracy(m, mh, x, xh):
    """per reduced mode, its poses' distance from the fp32-grade poses"""
    out = {}
    with torch.no_grad():
        engine.set_precision(m, 'fp32')
        y32 = m(x).double()
        engine.set_precision(m, 'tf32')
        yt = m(x).double()
        yh = mh(xh).double()
    engine.set_precision(m, 'fp32')
    for mode, y in (('tf32', yt), ('fp16', yh)):
        d = y - y32
        out[mode] = {'max_abs_dy': float(d.abs().max()), 'max_abs_y': float(y32.abs().max()),
                     'max_dy_over_max_y': float(d.abs().max() / y32.abs().max()),
                     'mean_joint_distance': float(d.norm(dim=-1).mean())}
    return out


def per_gemm(m, x, J, ch, fw, reps=5):
    """device ms of every GEMM launch of one forward, labelled (launch_times.gemm_shapes)"""
    with torch.no_grad():
        m(x)
    h = m.__dict__['_gast_handles'][('cuda', x.device.index)]
    lib = h.lib
    lib.gast_set_timing(h.h, 1)
    tot = None
    try:
        for _ in range(reps):
            with torch.no_grad():
                m(x)
            ms = (C.c_float * 512)()
            kinds = (C.c_int32 * 512)()
            n = lib.gast_get_timings(h.h, 512, ms, kinds)
            cur = [ms[i] for i in range(n)]
            tot = cur if tot is None else [a + b for a, b in zip(tot, cur)]
    finally:
        lib.gast_set_timing(h.h, 0)
    shapes = iter(gemm_shapes(x.shape[0], x.shape[1], J, ch, fw))
    out = []
    for i in range(n):
        if engine.LAUNCH_KINDS[kinds[i]].startswith('gemm'):
            layer, rows, N, K, epi = next(shapes)
            out.append((layer, rows, N, K, tot[i] / reps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--headline-only', action='store_true', help='only the alternated headline runs')
    ap.add_argument('--steps', type=int, default=20)
    args = ap.parse_args()
    emit({'card': card(), 'library': os.environ.get('GAST_B200_LIB', 'in-tree')})
    J, fw, ch = 17, [3, 3, 3], 128
    m = model(J, fw, ch)
    mh = copy.deepcopy(m).half()
    x = torch.from_numpy(synth.synth_input(4096, 27, J, 2, seed=5)).cuda()
    xh = x.half()
    for rnd in range(3):
        for prec in MODES:
            mm, xx = in_mode(m, mh, x, xh, prec)
            cps, ms = clips_per_s(mm, xx, args.steps)
            emit({'workload': 'headline 4096x27x17, 27-frame/128ch', 'round': rnd, 'precision': prec,
                  'clips_per_s': round(cps), 'ms_per_step': round(ms, 3)})
    emit(dict(workload='headline accuracy (synthetic weights)', **accuracy(m, mh, x, xh)))
    if args.headline_only:
        return
    for prec in MODES:
        mm, xx = in_mode(m, mh, x, xh, prec)
        rows = per_gemm(mm, xx, J, ch, fw)
        emit({'per_gemm_ms': prec, 'total_ms': round(sum(r[-1] for r in rows), 3),
              'gemms': [[r[0], r[1], r[2], r[3], round(r[4], 4)] for r in rows]})
    engine.set_precision(m, 'fp32')
    del mh, xh
    for name, (Jw, fww, chw, T, B) in (('81-frame/64ch 17-joint', (17, [3, 3, 3, 3], 64, 81, 2048)),
                                       ('27-frame/128ch 19-joint', (19, [3, 3, 3], 128, 27, 8192))):
        mw = model(Jw, fww, chw)
        mwh = copy.deepcopy(mw).half()
        xw = torch.from_numpy(synth.synth_input(B, T, Jw, 2, seed=5)).cuda()
        xwh = xw.half()
        for rnd in range(2):
            for prec in MODES:
                mm, xx = in_mode(mw, mwh, xw, xwh, prec)
                cps, ms = clips_per_s(mm, xx, args.steps)
                emit({'workload': '%s, %d clips' % (name, B), 'round': rnd, 'precision': prec,
                      'clips_per_s': round(cps), 'ms_per_step': round(ms, 3)})
        emit(dict(workload='%s accuracy (synthetic weights)' % name, **accuracy(mw, mwh, xw, xwh)))
        del mw, mwh, xw, xwh
    n = 1024
    frames = torch.from_numpy(synth.synth_input(n, 64, J, 2, seed=9)).cuda()
    for prec in ('fp32', 'tf32', 'fp32', 'tf32'):
        engine.set_precision(m, prec)
        ps = PoseStream(m, n)
        t = [0]

        def push():
            ps.push(frames[:, t[0] % 64])
            t[0] += 1
        ms1 = timed(push, 10, 100)
        ps = PoseStream(m, n)
        ms64 = timed(lambda: ps.push_frames(frames), 2, 10)
        emit({'workload': 'PoseStream 1024 streams, 27-frame/128ch', 'precision': prec,
              'push_ms': round(ms1, 4), 'frames_per_s_push': round(n / ms1 * 1e3),
              'push_frames_K64_ms': round(ms64, 3), 'frames_per_s_K64': round(n * 64 / ms64 * 1e3)})


if __name__ == '__main__':
    main()
