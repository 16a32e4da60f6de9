"""fp64 reference of the delayed stream (gast_b200.realtime.PoseStream, C ABI gast_stream_push_ex).

What a push must return is defined by the reference's inference helpers.  A stream's *sequence* is the frames pushed
from its start (construction or `reset`) up to its `end`.  Its poses are those of `UnchunkedGenerator(None, None,
[seq], pad, causal_shift, augment, ...)` followed by `tools/inference.evaluate` (tools/inference.py:19-41,
common/generators.py:210-233): edge padding of pad + causal_shift frames on the left and pad - causal_shift on the
right, the mirrored twin when augmenting, one forward, then un-flip and average.  Pose j of a sequence that started
with push t0 is returned by push t0 + j + latency (latency = pad - causal_shift), provided that push comes before the
stream's next reset.

`reference` builds exactly that.  It splits every stream at its resets and ends, independently of the library's
bookkeeping.  It pads each sequence and runs the dilated forward of the torch-CPU port (oracle/gast_torch_ref.py) in
float64, merges the twin, and maps each pose to the push that must return it.
"""
import functools
from collections import namedtuple

import numpy as np
import torch

from gast_b200 import synth
import kinkfree
import streamref as S

# J, filter widths (tuple), channels, streams, pushes, step counter before the first push, events, weight seed,
# causal, augment.  events: ((push index t, 'reset' | 'end', streams tuple or None for every stream), ...), applied
# in the listed order before push t.
Case = namedtuple('Case', 'J fw ch n T start events seed causal augment')

# left/right lists of tools/inference.py:14-15 (17 joints) and reconstruction.py:get_joints_info (19 joints; the
# keypoints use the same lists, reconstruction.py:185)
SYMMETRY = {
    17: ([4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]),
    19: ([5, 6, 7, 8, 13, 14, 15], [1, 2, 3, 4, 16, 17, 18]),
}


def symmetry(J):
    """(kps_left, kps_right, joints_left, joints_right) for J joints: the reference's lists, or a mirror pairing of
    joints 1..J-1 for the joint counts the reference has none for"""
    if J in SYMMETRY:
        left, right = SYMMETRY[J]
    else:
        k = (J - 1) // 2
        left, right = list(range(1, 1 + k)), list(range(1 + k, 1 + 2 * k))
    return left, right, left, right


def pad_shift(fw, causal):
    pad = (S.receptive_field(fw) - 1) // 2
    return pad, (pad if causal else 0)


def latency(fw, causal):
    pad, shift = pad_shift(fw, causal)
    return pad - shift


def module(case, dilated=False):
    """the drop-in model of `case` (Optimized1f, or the dilated SpatioTemporalModel with the same keys) with
    synthetic weights, in eval mode, on the CPU"""
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(case.J), [], []))
    cls = SpatioTemporalModel if dilated else SpatioTemporalModelOptimized1f
    m = cls(adj, case.J, 2, case.J, list(case.fw), causal=case.causal, dropout=0.05, channels=case.ch)
    synth.randomize_module(m, case.seed)
    return m.eval()


def frames(case):
    """the pushed keypoints (T, n, J, 2): frame t of every stream is pushed at push index t (rows of held pushes
    are ignored by the stream and never read here)"""
    return np.ascontiguousarray(synth.synth_input(case.n, case.T, case.J, 2, seed=100 + case.seed).transpose(1, 0, 2, 3))


def sequences(case, s):
    """[(t0, te, cut)]: the non-empty sequences of stream s.  Frames are pushed at t0 .. te-1; the pushes before
    `cut` (the next reset, or T) return its poses"""
    out = []
    t0, te = 0, None                          # te: push before which the sequence ended (None while live)
    for t in range(case.T + 1):
        for tt, kind, ss in case.events:
            if tt != t or not (ss is None or s in ss):
                continue
            if kind == 'end' and te is None:
                te = t
            elif kind == 'reset':
                out.append((t0, t if te is None else te, t))
                t0, te = t, None
    out.append((t0, case.T if te is None else te, case.T))
    return [(a, b, c) for a, b, c in out if b > a]


def expected_index(case, s):
    """(T,) int64: per push, the position within stream s's current sequence of the frame whose pose it returns,
    or -1"""
    lat = latency(case.fw, case.causal)
    idx = np.full(case.T, -1, dtype=np.int64)
    for t0, te, cut in sequences(case, s):
        for j in range(te - t0):
            if t0 + j + lat < cut:
                idx[t0 + j + lat] = j
    return idx


def generator_batch(seq, pad, shift, augment, kps_left, kps_right):
    """UnchunkedGenerator.next_epoch for one sequence (L, J, F) -> (1 or 2, L + 2 pad, J, F)"""
    b = np.pad(seq, ((pad + shift, pad - shift), (0, 0), (0, 0)), 'edge')[None]
    if augment:
        tw = b.copy()
        tw[0, :, :, 0] *= -1
        tw[0, :, kps_left + kps_right] = tw[0, :, kps_right + kps_left]
        b = np.concatenate([b, tw], axis=0)
    return b


def merge(pred, augment, joints_left, joints_right):
    """tools/inference.py:32-36: pred (1 or 2, L, J, 3) -> (L, J, 3)"""
    if not augment:
        return pred[0]
    q = pred[1].copy()
    q[:, :, 0] *= -1
    q[:, joints_left + joints_right] = q[:, joints_right + joints_left]
    return (pred[0] + q) / 2


def port(p, x, J, fw, causal):
    """the dilated forward of the port on padded sequences x (B, L + rf - 1, J, 2) in p's dtype -> (B, L, J, 3), in
    pieces of at most about S.FRAMES_PER_CALL input frames (each output frame sees exactly its own rf input frames)"""
    from oracle import gast_torch_ref as TR
    rf = S.receptive_field(fw)
    B, Tin = x.shape[:2]
    T = Tin - rf + 1
    bb = max(1, S.FRAMES_PER_CALL // (rf + 63))
    tc = max(64, S.FRAMES_PER_CALL // min(B, bb) - rf + 1)
    out = []
    for b0 in range(0, B, bb):
        xb = x[b0:b0 + bb]
        out.append(torch.cat([TR.forward(xb[:, a:min(T, a + tc) + rf - 1], p, kinkfree.masks(J), list(fw),
                                         causal=causal, strided=False) for a in range(0, T, tc)], dim=1))
    return torch.cat(out, dim=0)


def sequence_poses(seqs, J, fw, causal, augment, lists, state_dict, dtype=torch.float64):
    """[(L_k, J, 3)]: what UnchunkedGenerator + evaluate return for each sequence (L_k, J, 2) of `seqs`, by the
    port in `dtype` with the weights of `state_dict`"""
    pad, shift = pad_shift(fw, causal)
    kl, kr, jl, jr = lists
    p = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in state_dict.items()}
    out = [None] * len(seqs)
    groups = {}                                          # sequence length -> [k]: one batch each
    for k, sq in enumerate(seqs):
        groups.setdefault(len(sq), []).append(k)
    with torch.no_grad():
        for _, ks in sorted(groups.items()):
            b = np.concatenate([generator_batch(seqs[k], pad, shift, augment, kl, kr) for k in ks])
            got = port(p, torch.from_numpy(b).to(dtype), J, fw, causal).double().numpy()
            c = 2 if augment else 1
            for i, k in enumerate(ks):
                out[k] = merge(got[c * i:c * (i + 1)], augment, jl, jr)
    return out


def poses(case, x, streams, dtype=torch.float64, state_dict=None):
    """(y (len(streams), T, J, 3), index (len(streams), T)): per push, the pose the listed streams must return and
    the sequence position of its frame (-1 and NaN where nothing is due)"""
    lat = latency(case.fw, case.causal)
    sd = module(case).state_dict() if state_dict is None else state_dict
    y = np.full((len(streams), case.T, case.J, 3), np.nan)
    index = np.stack([expected_index(case, s) for s in streams])
    todo = [(i, t0, te, cut) for i, s in enumerate(streams) for t0, te, cut in sequences(case, s)]
    got = sequence_poses([x[t0:te, streams[i]] for i, t0, te, _ in todo], case.J, case.fw, case.causal, case.augment,
                         symmetry(case.J), sd, dtype)
    for (i, t0, te, cut), g in zip(todo, got):
        for j in range(te - t0):
            if t0 + j + lat < cut:
                y[i, t0 + j + lat] = g[j]
    return y, index


@functools.lru_cache(maxsize=None)
def reference(case, streams=None):
    """fp64 (poses, index) of the listed streams (every stream when None) for every push of `case`"""
    return poses(case, frames(case), tuple(range(case.n)) if streams is None else tuple(streams))


def errors(got, ref, index):
    """(max |got - ref| / max |ref|, relative L2 error) over the pushes that return a pose"""
    m = index >= 0
    return S.errors(np.asarray(got)[m], ref[m])
