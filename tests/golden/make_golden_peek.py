"""Peek goldens: what the UNMODIFIED reference returns for every prefix of a sequence, run on CPU fp32 with the set-up of
make_golden_delayed.py (`UnchunkedGenerator` + `tools.inference.evaluate`, or `reconstruction.evaluate` for 19 joints).

    python tests/golden/make_golden_peek.py

A live non-causal stream that has pushed the first l frames of a sequence and peeks K = latency frames must return the
poses of frames l - latency .. l - 1 of the sequence cut at frame l - 1: the reference's poses of the prefix x[:l],
whose right edge padding copies frame l - 1.  Writes tests/golden/peek_*.npz: x (T, J, 2) = the sequence,
prefixes (P,) = the prefix lengths l, y (P, latency, J, 3) = row k the pose of frame l - latency + k of prefix l (NaN
where that frame is before the sequence), and meta as for the delayed goldens.
"""
import numpy as np
import torch

from make_golden import SpatioTemporalModel, adj_for, keys_shapes, save, synth
from make_golden_delayed import SYM, reconstruction_evaluate


def peek_case(name, J, fw, ch, T, prefixes, augment, seed, xseed):
    from common.generators import UnchunkedGenerator
    m = SpatioTemporalModel(adj_for(J), J, 2, J, fw, causal=False, dropout=0.05, channels=ch)
    synth.randomize_module(m, seed)
    m.eval()
    rf = m.receptive_field()
    pad = (rf - 1) // 2
    left, right = SYM[J]
    x = synth.synth_input(1, T, J, 2, xseed)[0]
    prefixes = sorted(set(int(p) for p in prefixes))
    assert 1 <= prefixes[0] and prefixes[-1] <= T
    y = np.full((len(prefixes), pad, J, 3), np.nan, dtype=np.float32)
    for i, L in enumerate(prefixes):
        gen = UnchunkedGenerator(None, None, [x[:L]], pad=pad, causal_shift=0, augment=augment, kps_left=left,
                                 kps_right=right, joints_left=left, joints_right=right)
        if J == 17:
            from tools.inference import evaluate
            poses = evaluate(gen, m)[0]
        else:
            poses = reconstruction_evaluate()(gen, m, left, right, return_predictions=True)
        assert poses.shape == (L, J, 3)
        m_ = min(L, pad)
        y[i, pad - m_:] = poses[L - m_:]
    meta = dict(kind='peek', J=J, filter_widths=fw, channels=ch, causal=False, augment=augment, seed=seed,
                receptive_field=rf, pad=pad, latency=pad, kps_left=left, kps_right=right, joints_left=left,
                joints_right=right, keys=keys_shapes(m))
    save(name, x=x.astype(np.float32), prefixes=np.array(prefixes, dtype=np.int64), y=y, meta=meta)


def main():
    torch.manual_seed(0)
    # the reference's default 27-frame model at small width (latency 13): every prefix of 30 frames
    peek_case('peek_17_333_c32', 17, [3, 3, 3], 32, 30, range(1, 31), augment=False, seed=61, xseed=900)
    peek_case('peek_17_333_c32_aug', 17, [3, 3, 3], 32, 30, range(1, 31), augment=True, seed=62, xseed=910)
    # the 81-frame model (latency 40): prefixes around 1, pad and 2 pad
    peek_case('peek_17_3333_c64_aug', 17, [3, 3, 3, 3], 64, 90, [1, 2, 3, 39, 40, 41, 79, 80, 81, 90], augment=True,
              seed=63, xseed=920)
    peek_case('peek_19_333_c32_aug', 19, [3, 3, 3], 32, 30, [1, 5, 12, 13, 14, 20, 26, 27, 30], augment=True, seed=64,
              xseed=930)


if __name__ == '__main__':
    main()
