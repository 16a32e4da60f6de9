"""fp64 reference of the peek of a non-causal stream (gast_b200.realtime.PoseStream.peek, C ABI gast_stream_peek).

A peek of K frames returns what K more pushes would return if every stream's sequence ended at its newest frame.  So
it is defined by the reference's inference helpers on TRUNCATED sequences: a stream that has pushed frames t0 .. t-1 of
its current sequence (or all of it, when it ended before) peeks the poses of `UnchunkedGenerator([seq[:l]], pad, 0,
augment)` + `tools/inference.evaluate` (l = frames pushed), row k being the pose of frame t + k - t0 - latency where
that is one of the l frames.

Peek points are named by a push index t of a `delayedref.Case`: the peek is taken after pushes 0 .. t-1 and after the
events listed for push t (so a reset at t leaves nothing to peek and an end at t peeks the sequence's true tail), and
t = T is the peek after the last push.  The poses are computed by the port in float64 as in tests/delayedref.py;
pose j of a sequence only sees its own receptive field, so only the last min(l, latency) poses of each truncated
sequence are computed, from the input window they need.
"""
import numpy as np
import torch

import delayedref as D


def current(case, s, t):
    """(t0, te) of the sequence stream s is on at peek point t (te = case.T while it has not ended), or None"""
    cur = [(a, b) for a, b, c in D.sequences(case, s) if a <= t and (t < c or c == t == case.T)]
    return cur[-1] if cur else None


def expected_index(case, s, t, K):
    """(K,) int64: the sequence position of the frame of each row of stream s's peek at point t, or -1"""
    lat = D.latency(case.fw, case.causal)
    idx = np.full(K, -1, dtype=np.int64)
    cur = current(case, s, t)
    if cur is None:
        return idx
    t0, te = cur
    length = min(te, t) - t0
    j = t + np.arange(K) - t0 - lat
    ok = (j >= 0) & (j < length)
    idx[ok] = j[ok]
    return idx


def tail_poses(seqs, J, fw, augment, lists, state_dict, dtype=torch.float64):
    """[(min(L_k, latency), J, 3)]: the last min(L_k, latency) poses UnchunkedGenerator + evaluate return for each
    non-causal sequence (L_k, J, 2) of `seqs`, by the port in `dtype`"""
    pad, shift = D.pad_shift(fw, False)
    kl, kr, jl, jr = lists
    p = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in state_dict.items()}
    out = [None] * len(seqs)
    groups = {}                                          # poses wanted -> [k]: one batch each
    for k, sq in enumerate(seqs):
        groups.setdefault(min(len(sq), pad), []).append(k)
    with torch.no_grad():
        for m, ks in sorted(groups.items()):
            # the padded window of the last m poses: padded frames L - m .. L + 2 pad - 1
            b = np.concatenate([D.generator_batch(seqs[k], pad, shift, augment, kl, kr)[:, len(seqs[k]) - m:]
                                for k in ks])
            got = D.port(p, torch.from_numpy(b).to(dtype), J, fw, False).double().numpy()
            c = 2 if augment else 1
            for i, k in enumerate(ks):
                out[k] = D.merge(got[c * i:c * (i + 1)], augment, jl, jr)
    return out


def peeks(case, x, streams, points, K, state_dict=None, dtype=torch.float64):
    """(y (len(streams), len(points), K, J, 3), index (len(streams), len(points), K)): the peeks of K frames of the
    listed streams at the listed points, x (T, n, J, 2) the pushed frames (NaN where nothing is due)"""
    assert not case.causal
    lat = D.latency(case.fw, case.causal)
    sd = D.module(case).state_dict() if state_dict is None else state_dict
    index = np.stack([np.stack([expected_index(case, s, t, K) for t in points]) for s in streams])
    y = np.full(index.shape + (case.J, 3), np.nan)
    want = {}                                            # (stream, t0, frames pushed) -> truncated sequence
    for i, s in enumerate(streams):
        for q, t in enumerate(points):
            if (index[i, q] >= 0).any():
                t0, te = current(case, s, t)
                want[s, t0, min(te, t) - t0] = None
    keys = sorted(want)
    got = tail_poses([x[t0:t0 + n_, s] for s, t0, n_ in keys], case.J, case.fw, case.augment, D.symmetry(case.J), sd,
                     dtype)
    tails = dict(zip(keys, got))
    for i, s in enumerate(streams):
        for q, t in enumerate(points):
            rows = np.flatnonzero(index[i, q] >= 0)
            if rows.size:
                t0, te = current(case, s, t)
                length = min(te, t) - t0
                tail = tails[s, t0, length]              # poses of frames length - len(tail) .. length - 1
                y[i, q, rows] = tail[index[i, q, rows] - (length - len(tail))]
    return y, index


def errors(got, ref, index):
    """(max |got - ref| / max |ref|, relative L2 error) over the rows that return a pose"""
    return D.errors(got, ref, index)
