"""GPU: the cost of moving live streams between pools (PoseStream.export_streams / import_streams), and what it buys.

  * move: in a pool of 1024 streams that has pushed a few frames, export m = 1, 64 and 1024 streams and import them
    back into the same streams, against one lockstep single-frame push of the whole pool.  27-frame/128ch and
    81-frame/64ch non-causal models, augment off and on (2 library streams per stream).  Per call: the Python method's
    time on the stream from CUDA events around the call (median of REPS calls; at a few streams this is host time:
    the checks, allocations and the table copy, with the device waiting), and the C call's device time from REPS
    back-to-back calls between one event pair, with the bytes moved per direction (snapshot floats x 4 x library
    streams; each direction reads and writes them once) over it;
  * pools: a 1024-slot GraphedPoseStream ticking 64 active streams against the same 64 streams moved into a 64-slot
    GraphedPoseStream (27-frame/128ch, K = 1, no peek and a peek of `latency` frames): device ms per tick from events
    around each replay, and wall ms per tick over a window closed by a synchronise; and the one-off cost of the move.
Prints one JSON line per measurement, the first line with the card's name, power limit and SM clock read in the same
run.

    python tools/stream_move_bench.py [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
from chunk_stream_bench import card  # noqa: E402
from gast_b200 import engine, synth  # noqa: E402
from gast_b200.realtime import GraphedPoseStream, PoseStream  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f  # noqa: E402

REPS = 20
J = 17


def med(v):
    return sorted(v)[len(v) // 2]


def timed(fn, reps=REPS):
    """-> median device ms of fn() from an event pair around each call (after one untimed call)"""
    fn()
    out = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        out.append((a, b))
    torch.cuda.synchronize()
    return med([a.elapsed_time(b) for a, b in out])


def model(fw, ch):
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    m = SpatioTemporalModelOptimized1f(adj, J, 2, J, fw, causal=False, channels=ch, dropout=0.25)
    synth.randomize_module(m, 2)
    return m.cuda().eval()


def c_call_ms(ps, fn, sel, data, reps=REPS):
    """-> device ms per call of `reps` back-to-back C calls (gast_stream_export / _import) between one event pair:
    the library call without the Python method's checks and allocations"""
    h = engine.model_handle(ps.model, ps.device)
    lib = h.lib
    s = ps._lib_streams(sel).T.reshape(-1).astype(np.int32)
    c = np.full(s.size, max(ps.step, 1), dtype=np.int64)
    ws = torch.empty(int(lib.gast_stream_move_workspace_bytes(h.h, s.size)), dtype=torch.uint8, device=ps.device)
    st = torch.cuda.current_stream().cuda_stream
    args = (h.h, ps._state.data_ptr(), ps.copies * ps.n, s.ctypes.data, c.ctypes.data, s.size, data.data_ptr(),
            ws.data_ptr(), ws.numel(), st)
    assert getattr(lib, fn)(*args) == 0
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        getattr(lib, fn)(*args)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def move_costs(m, name, augment, emit):
    n = 1024
    ps = PoseStream(m, n, augment=augment)
    x = torch.from_numpy(synth.synth_input(n, 1, J, 2, seed=10)).cuda()[:, 0]
    for _ in range(3):
        ps.push(x)
    push_ms = timed(lambda: ps.push(x))
    for k in (1, 64, 1024):
        sel = list(range(0, n, n // k))[:k]
        snap = ps.export_streams(sel)
        exp_ms = timed(lambda: ps.export_streams(sel))
        imp_ms = timed(lambda: ps.import_streams(snap, sel))
        exp_c = c_call_ms(ps, 'gast_stream_export', sel, snap.data)
        imp_c = c_call_ms(ps, 'gast_stream_import', sel, snap.data)
        nbytes = snap.data.numel() * 4
        emit({'what': 'move', 'model': name, 'augment': augment, 'pool': n, 'streams': k, 'export_ms': exp_ms,
              'import_ms': imp_ms, 'export_c_ms': exp_c, 'import_c_ms': imp_c, 'lockstep_push_ms': push_ms,
              'bytes_per_direction': nbytes, 'export_c_GBps': 2 * nbytes / exp_c / 1e6,
              'import_c_GBps': 2 * nbytes / imp_c / 1e6})
        del snap
        torch.cuda.empty_cache()
    del ps
    torch.cuda.empty_cache()


def tick_costs(g, x, sel, ticks=100):
    """-> (device ms per tick around each replay, wall ms per tick) of push(x, streams=sel)"""
    spans = []
    replay = g.graph.replay

    def timed_replay():
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        replay()
        b.record()
        spans.append((a, b))
    g.graph.replay = timed_replay
    for _ in range(5):
        g.push(x, streams=sel)
    res = []
    for _ in range(3):
        spans.clear()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(ticks):
            g.push(x, streams=sel)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e3 / ticks
        res.append((sum(a.elapsed_time(b) for a, b in spans) / ticks, wall))
    g.graph.replay = replay
    return med([d for d, _ in res]), med([w for _, w in res])


def pool_costs(m, name, peek, emit):
    lat = (m.receptive_field() - 1) // 2
    P = lat if peek else 0
    big = GraphedPoseStream(m, 1024, K=1, peek=P)
    active = list(range(64))
    xb = torch.from_numpy(synth.synth_input(1024, 1, J, 2, seed=11)).cuda()
    for _ in range(3):
        big.push(xb, streams=active)
    big_dev, big_wall = tick_costs(big, xb, active)
    small = GraphedPoseStream(m, 64, K=1, peek=P)
    small.push(xb[:64], streams=[0])                     # the capture
    for _ in range(2):                                   # the second move is timed (the first loads the kernels)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        small.import_streams(big.export_streams(active), active)
        torch.cuda.synchronize()
        move_ms = (time.perf_counter() - t0) * 1e3
    small_dev, small_wall = tick_costs(small, xb[:64], None)
    emit({'what': 'pools', 'model': name, 'peek': P, 'active': 64,
          'pool1024_device_ms': big_dev, 'pool1024_wall_ms': big_wall,
          'pool64_device_ms': small_dev, 'pool64_wall_ms': small_wall, 'move_wall_ms': move_ms})
    del big, small
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', help='also append the JSON lines to this file')
    args = ap.parse_args()
    sink = open(args.out, 'a') if args.out else None

    def emit(rec):
        line = json.dumps(rec)
        print(line, flush=True)
        if sink:
            sink.write(line + '\n')
            sink.flush()
    emit({'card': card()})
    with torch.no_grad():
        for fw, ch in (([3, 3, 3], 128), ([3, 3, 3, 3], 64)):
            m = model(fw, ch)
            name = '%d-frame/%dch non-causal' % (m.receptive_field(), ch)
            for augment in (False, True):
                move_costs(m, name, augment, emit)
            if fw == [3, 3, 3]:
                for peek in (False, True):
                    pool_costs(m, name, peek, emit)
            del m
            torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
