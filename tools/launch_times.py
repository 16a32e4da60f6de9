"""GPU diagnostic: device time of every launch of one bench-workload forward, in launch order
(CUDA events inside the library: gast_set_timing / gast_get_timings).  Each GEMM launch is labelled with its
layer, rows, N, K and epilogue, and its rate is given as 3xTF32 TFLOP/s (6 rows N K / t: three products of
two flops per multiply-add), beside the card's name, power limit and SM clock read in the same run."""
import ctypes as C
import os
import subprocess
import sys
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
from gast_b200 import engine, synth  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModel  # noqa: E402


def gemm_shapes(B, T, J, ch, fw):
    """(layer, rows, N, K, epilogue) of every GEMM launch of the tensor-core forward, in launch order (gast_api.cu:
    run_block, run_stage).  T is the receptive field, so the dilated model runs the strided schedule (engine.py):
    the first stage keeps every fw[0]-th frame, each later stage every fw[i]-th."""
    def block(name, rows, C):
        return [(name + '.semch', rows, 2 * ((C + 63) // 64) * 128, C, 'semch'),   # both masks, 64 channels per tile
                (name + '.local_cat', rows, C, 2 * C, 'plain'),
                (name + '.global_g', rows, C, C, 'plain'),                        # 4 heads of C/4 channels
                (name + '.global_cat', rows, C, C, 'plain'),
                (name + '.block_cat', rows, 2 * C, 3 * C, 'plain')]
    Tp = (T - fw[0]) // fw[0] + 1
    out = block('block0', B * Tp * J, ch)
    for i in range(1, len(fw)):
        Cw = ch << i
        Tp = (Tp - fw[i]) // fw[i] + 1
        rows = B * Tp * J
        out += [('stage%d.conv' % i, rows, Cw, fw[i] * Cw, 'plain'), ('stage%d.1x1' % i, rows, Cw, Cw, 'plain')]
        out += block('block%d' % i, rows, Cw)
    return out


def card():
    d = {'name': torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.sm,clocks.max.sm',
                            '--format=csv,noheader,nounits'], capture_output=True, text=True, timeout=30)
        d['power_limit_w'], d['sm_mhz'], d['sm_max_mhz'] = [v.strip() for v in r.stdout.strip().split(',')]
    except (OSError, ValueError, subprocess.SubprocessError):
        pass
    return d


def main():
    # usage: launch_times.py [clips [joints [channels [filter,widths]]]]
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    J = int(sys.argv[2]) if len(sys.argv) > 2 else 17
    ch = int(sys.argv[3]) if len(sys.argv) > 3 else 128
    fw = [int(v) for v in sys.argv[4].split(',')] if len(sys.argv) > 4 else [3, 3, 3]
    T = 1
    for v in fw:
        T *= v
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    m = SpatioTemporalModel(adj, J, 2, J, fw, channels=ch)
    synth.randomize_module(m, 3)
    m = m.cuda().eval()
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=5)).cuda()
    with torch.no_grad():
        for _ in range(3):
            m(x)
    h = m.__dict__['_gast_handles'][('cuda', x.device.index)]
    lib = h.lib
    lib.gast_set_timing(h.h, 1)
    reps, tot = 5, None
    for _ in range(reps):
        with torch.no_grad():
            m(x)
        ms = (C.c_float * 512)()
        kinds = (C.c_int32 * 512)()
        n = lib.gast_get_timings(h.h, 512, ms, kinds)
        cur = [ms[i] for i in range(n)]
        tot = cur if tot is None else [a + b for a, b in zip(tot, cur)]
    lib.gast_set_timing(h.h, 0)
    print('card', card())
    names = [engine.LAUNCH_KINDS[kinds[i]] for i in range(n)]
    shapes = iter(gemm_shapes(B, T, J, ch, fw))
    gemm_ms = gemm_flop = 0.0
    for i in range(n):
        t = tot[i] / reps
        label = ''
        if names[i].startswith('gemm'):
            layer, rows, N, K, epi = next(shapes)
            assert names[i].endswith(epi), (names[i], layer)
            flop = 6.0 * rows * N * K
            gemm_ms += t
            gemm_flop += flop
            label = '%-18s rows %8d  N %4d  K %4d  %-5s %6.1f TFLOP/s' % (layer, rows, N, K, epi, flop / t * 1e-9)
        print('%2d %-16s %8.4f ms  %s' % (i, names[i], t, label))
    assert next(shapes, None) is None, 'fewer GEMM launches than the model has GEMMs'
    print('sum %.3f ms; GEMMs %.3f ms at %.1f TFLOP/s (3xTF32)' % (sum(tot) / reps, gemm_ms, gemm_flop / gemm_ms * 1e-9))


if __name__ == '__main__':
    main()
