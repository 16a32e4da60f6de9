"""The pass plan of the chunked eval-mode forward and backward (csrc/chunked.cuh, include/gast_b200.h), restated in
numpy: every output position is covered exactly once, every window reads inside [0, T) exactly the input frames its
outputs' receptive fields span, and one pass covers the call exactly when max_frames >= B * T_out."""
import numpy as np
import pytest


def out_frames(T, rf, strided):
    """gast_out_frames of a model with receptive field rf (odd filter widths: the strided output stride is rf)"""
    return T // rf if strided else T - rf + 1


def plan(B, T, rf, strided, max_frames):
    """[(b0, nb, t0, k, f0, Tin)]: clips [b0, b0+nb), output frames [t0, t0+k), input frames [f0, f0+Tin)"""
    T_out = out_frames(T, rf, strided)
    S = rf if strided else 1
    if T_out <= max_frames:
        clips = min(B, max_frames // T_out)
        return [(b0, min(clips, B - b0), 0, T_out, 0, T) for b0 in range(0, B, clips)]
    passes = []
    for b in range(B):
        for t0 in range(0, T_out, max_frames):
            k = min(max_frames, T_out - t0)
            passes.append((b, 1, t0, k, t0 * S, (k - 1) * S + rf))
    return passes


CASES = [  # B, T, rf, strided
    (1, 27, 27, False), (4, 27, 27, True), (3, 40, 27, False), (2, 100, 27, False), (5, 81, 27, True),
    (2, 300, 27, True), (3, 97, 81, False), (7, 243, 81, True), (1, 1000, 243, False), (6, 15, 15, False),
]


@pytest.mark.parametrize('B,T,rf,strided', CASES)
@pytest.mark.parametrize('max_frames', [1, 2, 3, 5, 13, 64, 1000])
def test_every_output_once_and_windows_inside(B, T, rf, strided, max_frames):
    T_out = out_frames(T, rf, strided)
    S = rf if strided else 1
    cover = np.zeros((B, T_out), np.int64)
    passes = plan(B, T, rf, strided, max_frames)
    for b0, nb, t0, k, f0, Tin in passes:
        assert 1 <= nb and 1 <= k and nb * k <= max_frames
        assert 0 <= f0 and f0 + Tin <= T
        # the window is an ordinary call on Tin frames: it gives exactly its k outputs
        assert out_frames(Tin, rf, strided) == k
        # it holds the frames the receptive fields of its outputs span: a window exactly those, whole clips all of T
        reads = set()
        for t in range(t0, t0 + k):
            reads.update(range(t * S, t * S + rf))
        if Tin < T:
            assert min(reads) == f0 and max(reads) + 1 == f0 + Tin
        else:
            assert f0 == 0 and max(reads) < T
        cover[b0:b0 + nb, t0:t0 + k] += 1
    assert (cover == 1).all()
    assert (len(passes) == 1) == (max_frames >= B * T_out)
    # passes run clip by clip, window by window
    assert passes == sorted(passes)


@pytest.mark.parametrize('B,T,rf,strided', CASES)
def test_largest_pass_does_not_depend_on_T_or_B(B, T, rf, strided):
    """the workspace follows the largest pass: with windows its input length depends on max_frames and rf only, and
    with whole clips on the clips per pass only once B fills a pass"""
    T_out = out_frames(T, rf, strided)
    S = rf if strided else 1
    for max_frames in (1, 3, 16):
        if T_out > max_frames:
            for T2 in (T + S, T + 7 * S, 4 * T):
                big = max(p[5] for p in plan(B, T2, rf, strided, max_frames))
                assert big == (max_frames - 1) * S + rf
        else:
            clips = max_frames // T_out
            for B2 in (clips, clips + 1, 3 * clips + 2):
                assert max(p[1] for p in plan(B2, T, rf, strided, max_frames)) == clips
