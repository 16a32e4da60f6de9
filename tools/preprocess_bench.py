"""GPU: what the video demo's keypoint repair and person placement cost on the host (the numpy restatement, bit-identical
to the reference: tests/preprocessref.py) and on the device (device.tools.preprocess).  Wall-clock ms per call, with a
device synchronise around each timed window and a warm-up first.
  - offline: two persons x 50k frames through h36m_coco_format -> revise_kpts -> revise_skes.  The host side starts
    from numpy arrays, the device side from CUDA tensors (the predictions already on the device, as gen_pose leaves
    them); the device chain includes h36m_coco_format's one host read.
  - per tick, M = 1, 64, 1024 persons: revise_skes_real_time on numpy arrays against CUDA tensors.
Prints one JSON line per measurement, the first with the card's name, power limit and SM clock read in the same run.

    python tools/preprocess_bench.py
"""
import json
import os
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
sys.path.insert(0, os.path.join(REPO, 'tests'))
from chunk_stream_bench import card  # noqa: E402
import preprocessref as R  # noqa: E402
import device.tools.preprocess as D  # noqa: E402


def wall_ms(fn, warm, reps):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def offline_inputs(T, seed=0):
    rs = np.random.RandomState(seed)
    kp = rs.uniform(0, 1900, (2, T, 17, 2)).astype(np.float32)
    sc = rs.uniform(0.0, 1.0, (2, T, 17)).astype(np.float32)
    sc[..., [2, 3, 5, 6]] = rs.uniform(0.2, 0.4, (2, T, 4)).astype(np.float32)
    kp[0, int(0.8 * T):] = 0
    kp[1, :int(0.2 * T)] = 0
    return kp, sc


def main():
    print(json.dumps({'card': card()}), flush=True)
    T = 50_000
    kp, sc = offline_inputs(T)
    _, _, vf = R.h36m_coco_format(kp, sc)
    rs = np.random.RandomState(1)
    pred = [rs.standard_normal((len(f), 17, 3)).astype(np.float32) for f in vf]

    def host():
        hk, hs, f = R.h36m_coco_format(kp, sc)
        return R.revise_skes(pred, R.revise_kpts(hk, hs, f), f)

    dkp, dsc = torch.from_numpy(kp).cuda(), torch.from_numpy(sc).cuda()
    dpred = [torch.from_numpy(p).cuda() for p in pred]

    def dev():
        hk, hs, f = D.h36m_coco_format(dkp, dsc)
        return D.revise_skes(dpred, D.revise_kpts(hk, hs, f), f)

    assert np.array_equal(dev().cpu().numpy(), host())
    h_ms, d_ms = wall_ms(host, 1, 3), wall_ms(dev, 3, 20)
    print(json.dumps({'what': 'offline h36m_coco_format -> revise_kpts -> revise_skes', 'persons': 2, 'frames': T,
                      'host_numpy_ms': h_ms, 'device_ms': d_ms, 'host_over_device': h_ms / d_ms}), flush=True)
    for M in (1, 64, 1024):
        p = rs.standard_normal((M, 17, 3)).astype(np.float32)
        k = rs.uniform(0, 1920, (M, 17, 2)).astype(np.float32)
        dp, dk = torch.from_numpy(p).cuda(), torch.from_numpy(k).cuda()
        assert np.array_equal(D.revise_skes_real_time(dp, dk, 1920).cpu().numpy(), R.revise_skes_real_time(p, k, 1920))
        h_ms = wall_ms(lambda: R.revise_skes_real_time(p, k, 1920), 10, 200)
        d_ms = wall_ms(lambda: D.revise_skes_real_time(dp, dk, 1920), 10, 200)
        print(json.dumps({'what': 'per tick revise_skes_real_time', 'persons': M, 'host_numpy_ms': h_ms,
                          'device_ms': d_ms, 'host_over_device': h_ms / d_ms}), flush=True)


if __name__ == '__main__':
    main()
