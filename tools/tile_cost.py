"""GPU diagnostic: what one 128 x 128 output tile of the tensor-core GEMM core costs, split into a fixed part and a
part per 32-wide K stage.

Times gast_debug_gemm (core 0, plain epilogue) with CUDA events at the block-0 row count of the headline forward
(626,688 rows = 4096 clips x 9 frames x 17 joints) for N = 128 and 512 and K = 128 .. 1536, and fits the time a
tile occupies an SM,

    t * SMs / tiles = a + b * stages,   stages = K / 32,

by least squares over the K sweep of each N.  `a` is what a tile costs however short its K loop is (launch, set-up,
first ring fill, epilogue, whatever the K loop cannot hide); `b` is the cost of one ring stage.  Each shape is also
given as 3xTF32 TFLOP/s (6 M N K / t) and with the A bytes it needs from HBM in two tile orders (computed, not
measured): every column tile re-reading its rows (`A x col tiles`) or a row tile's column tiles adjacent (`A once`).
The card's name, power limit and SM clock are read in the same run."""
import ctypes as C
import os
import sys

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
from gast_b200 import _lib  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from launch_times import card  # noqa: E402

M = 626688
NS = (128, 512)
KS = (128, 256, 384, 768, 1536)


def time_gemm(lib, a, w, o, N, K, reps):
    ms = C.c_float(0.0)
    st = torch.cuda.current_stream().cuda_stream
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, 0, 0, None, st)   # warm-up
    assert rc == 0, _lib.last_error()
    rc = lib.gast_debug_gemm(a.data_ptr(), w.data_ptr(), o.data_ptr(), M, N, K, 0, 0, reps, C.byref(ms), st)
    assert rc == 0, _lib.last_error()
    return ms.value


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    lib = _lib.load()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device='cuda').manual_seed(7)
    abuf = torch.randn(M * max(KS), device='cuda', generator=g)
    wbuf = torch.randn(max(NS) * max(KS), device='cuda', generator=g) * 0.05
    obuf = torch.empty(M * max(NS), device='cuda')
    print('card', card(), 'SMs', sms)
    print('%5s %5s %7s %6s %9s %10s %8s %12s %9s' % ('N', 'K', 'stages', 'tiles', 'ms', 'us/tile/SM', 'TFLOP/s',
                                                    'A x coltiles', 'A once'))
    for N in NS:
        st, per = [], []
        for K in KS:
            t = time_gemm(lib, abuf[:M * K], wbuf[:N * K], obuf[:M * N], N, K, reps)
            row_tiles, col_tiles = (M + 127) // 128, (N + 127) // 128
            tiles = row_tiles * col_tiles
            per_tile = t * 1e3 * sms / tiles
            abytes = M * K * 4
            st.append(K // 32)
            per.append(per_tile)
            print('%5d %5d %7d %6d %9.3f %10.3f %8.1f %10.2f GB %6.2f GB' % (
                N, K, K // 32, tiles, t, per_tile, 6.0 * M * N * K / t * 1e-9, abytes * col_tiles * 1e-9,
                abytes * 1e-9))
        b, a = np.polyfit(np.array(st, dtype=np.float64), np.array(per, dtype=np.float64), 1)
        print('N %d: per tile = %.3f us + %.4f us x stages; fixed part %.0f %% of a K = 128 tile, %.0f %% at K = 256'
              % (N, a, b, 100 * a / (a + 4 * b), 100 * a / (a + 8 * b)))
    print('card after', card())


if __name__ == '__main__':
    main()
