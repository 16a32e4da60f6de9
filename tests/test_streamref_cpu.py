"""The fp64 per-frame stream reference of tests/streamref.py, on the CPU: it reproduces the reference's own per-frame
outputs (the stream_* goldens, made by the unmodified UnchunkedGenerator(pad, causal_shift=pad) + causal
SpatioTemporalModel in fp32), and its split at resets equals recomputing each frame from its own window."""
import numpy as np
import pytest
import torch

from conftest import load_golden
import streamref as S

# max |y_golden - y64| / max |y64| measured over the three goldens: 1.7e-6, 1.9e-6 and 2.1e-6 (the reference's fp32
# rounding; the fp32 port reproduces the goldens to the last bit on a single-socket x86 host)
GOLDEN_BAR = 1e-5


@pytest.mark.parametrize('name', ['stream_17_333_c32_causal', 'stream_17_333_c128_causal', 'stream_17_3333_c64_causal'])
def test_reference_matches_stream_goldens(name):
    g = load_golden(name)
    meta = g['meta']
    n, T = g['x'].shape[:2]
    case = S.Case(meta['J'], tuple(meta['filter_widths']), meta['channels'], n, T, 0, (), meta['seed'])
    assert S.receptive_field(case.fw) == meta['receptive_field']
    x = np.ascontiguousarray(g['x'].transpose(1, 0, 2, 3))                    # (T, n, J, 2): push order
    y64 = S.poses(case, x, tuple(range(n)))
    mx, l2 = S.errors(g['y'], y64)
    assert mx <= GOLDEN_BAR and l2 <= GOLDEN_BAR, (mx, l2)
    y32 = S.poses(case, x, tuple(range(n)), dtype=torch.float32)
    assert np.abs(y32 - g['y']).max() <= 1e-6 * np.abs(g['y']).max()


def test_reset_segments_equal_per_frame_windows():
    """a stream's pose at push t is the causal forward of its last rf frames since its latest reset, the frames
    before that reset replaced by copies of the reset frame"""
    case = S.Case(17, (3, 3), 16, 3, 14, 0, ((4, (1,)), (5, (1,)), (9, None), (13, (2,))), 8)
    rf = S.receptive_field(case.fw)
    x = S.frames(case)
    y = S.reference(case)
    p = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in S.module(case).state_dict().items()}
    for s in range(case.n):
        for t in range(case.T):
            t0 = max(t0 for t0, _ in S.segments(case, s) if t0 <= t)
            hist = x[t0:t + 1, s]
            window = np.concatenate([np.repeat(hist[:1], max(0, rf - len(hist)), axis=0), hist[-rf:]])
            with torch.no_grad():
                want = S.port_causal(p, torch.from_numpy(window[None]).double(), case.J, case.fw)[0, -1].numpy()
            assert np.abs(y[s, t] - want).max() <= 1e-12, (s, t)
