"""numpy model of the stream state layout (stream_plan in csrc/stream.cuh) and of moving streams between states
(gast_stream_export / gast_stream_import, include/gast_b200.h).

A state of n streams is, after its 256-byte aligned base, the input history xhist (n, k0, J, F) and per temporal
stage i = 1 .. L-1 a ring (R_i, n, J, C_i), each part starting at a multiple of 64 floats.  A stream at count c keeps
the stage input of time t in slot t mod R_i, so its slots hold times c - R_i .. c - 1.  Its snapshot is its input
history, then every ring in time order (oldest first)."""
import numpy as np


def parts(J, F, fw, ch):
    """[(R, row floats)] of one stream: the input history as one row, then every ring"""
    out, d = [(1, fw[0] * J * F)], fw[0]
    for i in range(1, len(fw)):
        out.append((fw[i] * d, J * (ch << i)))
        d *= fw[i]
    return out


def snapshot_floats(J, F, fw, ch):
    return sum(R * row for R, row in parts(J, F, fw, ch))


def layout(J, F, fw, ch, n):
    """([(state offset, R, row floats)] of the parts, state floats): offsets in floats from the aligned base"""
    off, out = 0, []
    for R, row in parts(J, F, fw, ch):
        nf = R * n * row
        out.append((off, R, row))
        off += (nf + 63) & ~63
    return out, off


def state_index(J, F, fw, ch, n, s, count):
    """(snapshot floats,) int64: the state float each snapshot float of stream s at `count` sits in"""
    idx = []
    for q, (off, R, row) in enumerate(layout(J, F, fw, ch, n)[0]):
        if q == 0:                                           # (n, k0 J F): one time-ordered row per stream
            idx.append(off + s * row + np.arange(row))
            continue
        slots = (count + np.arange(R)) % R                   # (c - R + j) mod R: oldest first
        idx.append((off + (slots[:, None] * n + s) * row + np.arange(row)[None, :]).reshape(-1))
    return np.concatenate(idx).astype(np.int64)


def export(state, J, F, fw, ch, n, streams, counts):
    """state (state floats,) -> (m, snapshot floats): the snapshots of the listed streams at their counts"""
    return np.stack([state[state_index(J, F, fw, ch, n, s, c)] for s, c in zip(streams, counts)])


def import_(state, J, F, fw, ch, n, streams, counts, snap):
    """-> a copy of state with snapshot snap[i] written to stream streams[i] at count counts[i]"""
    out = state.copy()
    for s, c, row in zip(streams, counts, snap):
        out[state_index(J, F, fw, ch, n, s, c)] = row
    return out
