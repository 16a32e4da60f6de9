"""Scoring a lifted test set on the device, the way the reference reports it (trainval.py:304-328 run_evaluation ->
main.py:299-353 evaluate per action; common/loss.py:56-90 pck / auc for MPI-INF-3DHP-style numbers).

`evaluate_sequences` lifts every sequence with `realtime.lift_sequences` (bounded memory, the reference's TTA merge),
scores all of them with ONE `gast_pose_metrics` launch pair over the concatenated poses (one row per sequence), copies
the rows to the host once, and adds them into their groups there in double.  The reference instead runs one forward
per sequence, syncs on `.item()` per sequence and runs p_mpjpe as a float32 numpy SVD on the host.
"""
import numpy as np
import torch

from . import pipeline as _P
from .engine import GastError
from .realtime import lift_sequences

AUC_THRESHOLDS = torch.linspace(0, 150, 31).tolist()     # common/loss.py:83, mpii_compute_3d_pck.m's range
PCK_THRESHOLD = 150.0                                    # common/loss.py:76, pck's default


class GroupScore(object):
    """The scores of one group, in the poses' units (main.evaluate's e1 / e2 are mpjpe / p_mpjpe times 1000):
    frames; mpjpe and p_mpjpe, the means over the group's frames (main.evaluate's N-weighted sums over its sequences);
    per_joint (J,) the mean distance of each joint; with thresholds, pck at 150, auc over the 31 thresholds of
    common/loss.auc and pck_at {threshold: fraction} for the thresholds asked for.  NaN when the group has no frames."""

    def __init__(self, row, J, thresholds, procrustes):
        f = float(row[0])
        with np.errstate(divide='ignore', invalid='ignore'):
            self.frames = int(f)
            self.mpjpe = row[1] / f if f > 0 else float('nan')
            self.p_mpjpe = row[2] / f if f > 0 and procrustes else float('nan')
            self.per_joint = row[3:3 + J] / f if f > 0 else np.full(J, np.nan)
        self.pck = self.auc = self.pck_at = None
        if thresholds is not None:
            n = f * J
            frac = [c / n if n > 0 else float('nan') for c in row[3 + J:].tolist()]
            grid = frac[:len(AUC_THRESHOLDS)]
            self.pck = grid[AUC_THRESHOLDS.index(PCK_THRESHOLD)]
            self.auc = torch.tensor(grid, dtype=torch.float64).mean().item()
            self.pck_at = dict(zip(thresholds, frac[len(AUC_THRESHOLDS):]))

    def __repr__(self):
        return 'GroupScore(frames=%d, mpjpe=%.6g, p_mpjpe=%.6g)' % (self.frames, self.mpjpe, self.p_mpjpe)


class Evaluation(object):
    """`groups`: the labels in first-seen order; `scores[label]` (also `result[label]`) a GroupScore."""

    def __init__(self, groups, scores):
        self.groups = groups
        self.scores = scores

    def __getitem__(self, label):
        return self.scores[label]

    def action_wise(self):
        """(mean over groups of mpjpe, of p_mpjpe): run_evaluation's 'action-wise average' (trainval.py:327-328),
        in the poses' units"""
        return (float(np.mean([self.scores[g].mpjpe for g in self.groups])),
                float(np.mean([self.scores[g].p_mpjpe for g in self.groups])))


def evaluate_sequences(model_pos, poses_2d, poses_3d, groups=None, augment=False, kps_left=None, kps_right=None,
                       joints_left=None, joints_right=None, procrustes=True, thresholds=None, zero_root=True,
                       n_streams=64, chunk=256):
    """Score a test set by group.  poses_2d[i] (T_i, J_in, F) and poses_3d[i] (T_i, J_out, 3), as fetch_actions builds
    them (numpy or tensors); groups[i] any hashable label (default: one group, None).  The poses are what
    `UnchunkedGenerator` + the model (+ the TTA merge with augment=True) give, lifted by `lift_sequences` (every one of
    its restrictions applies: a half model is refused before any launch).  zero_root scores against targets whose
    joint 0 is 0 (main.py:327), without writing the caller's arrays.  thresholds: None for no PCK; True for pck at
    150 and auc; or a sequence of thresholds, whose fractions are reported in pck_at besides.  A group's scores depend
    only on its own sequences.  Returns an Evaluation."""
    n = len(poses_2d)
    if len(poses_3d) != n or (groups is not None and len(groups) != n):
        raise GastError('evaluate_sequences: %d 2D sequences, %d 3D sequences and %s group labels'
                        % (n, len(poses_3d), 'no' if groups is None else len(groups)))
    lengths = [int(p.shape[0]) for p in poses_2d]
    J = int(model_pos.num_joints_out)
    for i, p in enumerate(poses_3d):
        if tuple(p.shape) != (lengths[i], J, 3):
            raise GastError('evaluate_sequences: poses_3d[%d] must be (%d, %d, 3), got %s'
                            % (i, lengths[i], J, tuple(p.shape)))
    extra = [] if thresholds is None or thresholds is True else [float(t) for t in thresholds]
    thr = AUC_THRESHOLDS + extra if thresholds is not None else []
    preds = lift_sequences(model_pos, poses_2d, n_streams=n_streams, chunk=chunk, augment=augment, kps_left=kps_left,
                           kps_right=kps_right, joints_left=joints_left, joints_right=joints_right)
    dev = next(model_pos.parameters()).device
    pred = torch.cat(preds) if n else torch.empty((0, J, 3), dtype=torch.float32, device=dev)
    if all(isinstance(p, torch.Tensor) for p in poses_3d):
        tgt = torch.cat([p.to(device=dev, dtype=torch.float32) for p in poses_3d]) if n else torch.empty_like(pred)
    else:                                                 # one upload of the concatenated host arrays
        tgt = torch.as_tensor(np.concatenate([np.asarray(p, dtype=np.float32) for p in poses_3d])).to(dev)
    seg = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    rows = _P.pose_metrics(pred, tgt, seg, thr, zero_root=zero_root, procrustes=procrustes).cpu().numpy() if n \
        else np.zeros((0, 3 + J + len(thr)))
    labels = [None] * n if groups is None else list(groups)
    order, acc = [], {}
    for lab, r in zip(labels, rows):
        if lab not in acc:
            order.append(lab)
            acc[lab] = np.zeros_like(r)
        acc[lab] += r
    if not order:
        order, acc[None] = [None], np.zeros(3 + J + len(thr))
    return Evaluation(order, {g: GroupScore(acc[g], J, extra if thresholds is not None else None, procrustes)
                              for g in order})
