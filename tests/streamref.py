"""fp64 per-frame reference of the O(1) causal stream (gast_b200.realtime.CausalStream, C ABI gast_stream_push).

What a push must return is defined by the reference's real-time path: for every frame, the whole-sequence causal
forward of the stream so far, left-padded with rf - 1 copies of the stream's first frame (UnchunkedGenerator(pad,
causal_shift=pad), common/generators.py:210-221).  A reset starts a new sequence on that stream at the frame pushed
next.  `reference` builds exactly that: it splits every stream at its resets, edge-pads each segment on the left and
runs the dilated causal forward of the torch-CPU port (oracle/gast_torch_ref.py) on it in float64.  The result is
one pose per pushed frame, independent of the ring geometry, the step counter and the GEMM core.
"""
import functools
from collections import namedtuple

import numpy as np
import torch

from gast_b200 import synth
import kinkfree

# J, filter widths (tuple), channels, streams, pushes, step counter before the first push, resets, weight seed.
# resets: ((push index t, streams tuple or None for every stream), ...): those streams start anew with frame t.
Case = namedtuple('Case', 'J fw ch n T start resets seed')

FRAMES_PER_CALL = 6000      # batch * window frames per port call: bounds the memory of the attention materialisation


def receptive_field(fw):
    return int(np.prod(fw))


def module(case, dilated=False):
    """the drop-in causal model of `case` (Optimized1f, or the dilated SpatioTemporalModel with the same keys) with
    synthetic weights, in eval mode, on the CPU"""
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(case.J), [], []))
    cls = SpatioTemporalModel if dilated else SpatioTemporalModelOptimized1f
    m = cls(adj, case.J, 2, case.J, list(case.fw), causal=True, dropout=0.05, channels=case.ch)
    synth.randomize_module(m, case.seed)
    return m.eval()


def frames(case):
    """the pushed keypoints (T, n, J, 2): frame t of every stream is pushed at push index t"""
    return np.ascontiguousarray(synth.synth_input(case.n, case.T, case.J, 2, seed=100 + case.seed).transpose(1, 0, 2, 3))


def segments(case, s):
    """[(t0, t1), ...]: the push ranges of stream s between its resets"""
    starts = {0} | {t for t, ss in case.resets if ss is None or s in ss}
    starts = sorted(t for t in starts if t < case.T)
    return list(zip(starts, starts[1:] + [case.T]))


def padded(seg, rf):
    """seg (L, J, F) -> (L + rf - 1, J, F): the causal edge padding of UnchunkedGenerator(pad, causal_shift=pad)"""
    return np.concatenate([np.repeat(seg[:1], rf - 1, axis=0), seg], axis=0)


def port_causal(p, x, J, fw):
    """the dilated causal forward of the port on x (B, T + rf - 1, J, 2) in p's dtype -> (B, T, J, 3), in pieces of
    at most about FRAMES_PER_CALL input frames (each output frame sees exactly its own rf input frames either way)"""
    from oracle import gast_torch_ref as TR
    rf = receptive_field(fw)
    B, Tin = x.shape[:2]
    T = Tin - rf + 1
    bb = max(1, FRAMES_PER_CALL // (rf + 63))                     # streams per call
    tc = max(64, FRAMES_PER_CALL // min(B, bb) - rf + 1)          # output frames per call
    out = []
    for b0 in range(0, B, bb):
        xb = x[b0:b0 + bb]
        out.append(torch.cat([TR.forward(xb[:, a:min(T, a + tc) + rf - 1], p, kinkfree.masks(J), list(fw),
                                         causal=True, strided=False) for a in range(0, T, tc)], dim=1))
    return torch.cat(out, dim=0)


def poses(case, x, streams, dtype=torch.float64, state_dict=None):
    """the poses (len(streams), T, J, 3) that pushing x (T, n, J, 2) frame by frame must return for the listed
    streams, by the port in `dtype`, with the weights of `state_dict` (default: those of module(case))"""
    rf = receptive_field(case.fw)
    sd = module(case).state_dict() if state_dict is None else state_dict
    p = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in sd.items()}
    y = np.zeros((len(streams), x.shape[0], case.J, 3))
    groups = {}                                          # segment length -> [(row, stream, t0, t1)]: one batch each
    for i, s in enumerate(streams):
        for t0, t1 in segments(case, s):
            groups.setdefault(t1 - t0, []).append((i, s, t0, t1))
    with torch.no_grad():
        for L, segs in sorted(groups.items()):
            xs = np.stack([padded(x[t0:t1, s], rf) for _, s, t0, t1 in segs])
            got = port_causal(p, torch.from_numpy(xs).to(dtype), case.J, case.fw).double().numpy()
            for (i, _, t0, t1), g in zip(segs, got):
                y[i, t0:t1] = g
    return y


@functools.lru_cache(maxsize=None)
def reference(case, streams=None):
    """fp64 poses (len(streams), T, J, 3) of the listed streams (every stream when None) for every push of `case`"""
    return poses(case, frames(case), tuple(range(case.n)) if streams is None else tuple(streams))


def errors(got, ref):
    """(max |got - ref| / max |ref|, relative L2 error) of poses against the fp64 reference"""
    got = np.asarray(got, dtype=np.float64)
    return (float(np.abs(got - ref).max() / np.abs(ref).max()),
            float(np.linalg.norm(got - ref) / np.linalg.norm(ref)))
