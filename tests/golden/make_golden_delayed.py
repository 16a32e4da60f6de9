"""Delayed-stream goldens: run the UNMODIFIED reference (as tests/golden/make_golden.py does, whose set-up and helpers
this script reuses) on CPU fp32 the way its inference helpers run a model on whole sequences:
`UnchunkedGenerator(None, None, seqs, pad, causal_shift, augment, kps_left, kps_right, joints_left, joints_right)`
(common/generators.py:162-236) followed by `tools.inference.evaluate` (tools/inference.py:19-41: one forward per
sequence, un-flip and average the mirrored twin), or for 19 joints by `reconstruction.evaluate`, which un-flips with
the 19-joint lists.

    python tests/golden/make_golden_delayed.py

Writes tests/golden/delayed_*.npz: x = the sequences concatenated along time (sum L, J, 2), y = the poses
concatenated the same way (sum L, J, 3), and meta (lengths, model, padding, symmetry lists).  A stream that pushes
sequence k and then ends it must return y of sequence k.  Weights are re-created from `gast_b200.synth`, as for every
golden.
"""
import sys
import types

import numpy as np
import torch

from make_golden import SpatioTemporalModel, adj_for, keys_shapes, save, synth

# tools/inference.py:14-15 and reconstruction.py:get_joints_info (reconstruction.py:185: kps lists = joints lists)
SYM = {17: ([4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]),
       19: ([5, 6, 7, 8, 13, 14, 15], [1, 2, 3, 4, 16, 17, 18])}


def reconstruction_evaluate():
    """reconstruction.evaluate (reconstruction.py:148-170), the whole-sequence helper of the reference's 19-joint
    path: tools.inference.evaluate un-flips with the 17-joint lists of its module.  reconstruction.py imports cv2 and
    the matplotlib renderer at module level; neither is used by `evaluate` nor installed here, so both are stubbed
    (as make_golden.py stubs torchsummary)."""
    sys.modules.setdefault('cv2', types.SimpleNamespace())
    sys.modules.setdefault('tools.visualization', types.SimpleNamespace(render_animation=None))
    import reconstruction
    return reconstruction.evaluate


def delayed_case(name, J, fw, ch, lengths, causal, augment, seed, xseed):
    from common.generators import UnchunkedGenerator
    m = SpatioTemporalModel(adj_for(J), J, 2, J, fw, causal=causal, dropout=0.05, channels=ch)
    synth.randomize_module(m, seed)
    m.eval()
    rf = m.receptive_field()
    pad = (rf - 1) // 2
    shift = pad if causal else 0
    left, right = SYM[J]
    seqs = [synth.synth_input(1, L, J, 2, xseed + k)[0] for k, L in enumerate(lengths)]
    gen = UnchunkedGenerator(None, None, seqs, pad=pad, causal_shift=shift, augment=augment, kps_left=left,
                             kps_right=right, joints_left=left, joints_right=right)
    if J == 17:
        from tools.inference import evaluate
        ys = evaluate(gen, m)
    else:
        assert len(lengths) == 1                     # reconstruction.evaluate returns the first sequence's poses
        ys = [reconstruction_evaluate()(gen, m, left, right, return_predictions=True)]
    assert [y.shape for y in ys] == [(L, J, 3) for L in lengths]
    meta = dict(kind='delayed', J=J, filter_widths=fw, channels=ch, causal=causal, augment=augment, seed=seed,
                lengths=list(lengths), receptive_field=rf, pad=pad, causal_shift=shift, kps_left=left, kps_right=right,
                joints_left=left, joints_right=right, keys=keys_shapes(m))
    save(name, x=np.concatenate(seqs).astype(np.float32), y=np.concatenate(ys).astype(np.float32), meta=meta)


def main():
    torch.manual_seed(0)
    # the reference's default (non-causal) models, load_model_layer / reconstruction.py, at small width
    delayed_case('delayed_17_333_c32', 17, [3, 3, 3], 32, [45, 30], causal=False, augment=False, seed=21, xseed=800)
    # two sequences, the second shorter than pad = 13
    delayed_case('delayed_17_333_c32_aug', 17, [3, 3, 3], 32, [40, 9], causal=False, augment=True, seed=22, xseed=810)
    delayed_case('delayed_17_3333_c64_aug', 17, [3, 3, 3, 3], 64, [100], causal=False, augment=True, seed=23,
                 xseed=820)
    # the reference's real-time model (27 frames, 128 channels, causal) run the way its helpers run it
    delayed_case('delayed_17_333_c128_causal_aug', 17, [3, 3, 3], 128, [50], causal=True, augment=True, seed=24,
                 xseed=830)
    delayed_case('delayed_19_333_c32_aug', 19, [3, 3, 3], 32, [35], causal=False, augment=True, seed=25, xseed=840)


if __name__ == '__main__':
    main()
