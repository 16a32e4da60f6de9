"""Golden outputs of the video demo's keypoint repair and person placement from the UNMODIFIED reference
(tools/preprocess.py: load_json, h36m_coco_format, revise_kpts, revise_skes, revise_skes_real_time; tools/inference.py:
gen_pose with a small seeded 27-frame, 16-channel model).

Run in the build container only (the GPU box has no reference checkout):
    python tests/golden/make_golden_preprocess.py
Writes tests/golden/preprocess_17.npz (and nothing else).  The model's weights are re-created from `gen_pose_seed` by
gast_b200.synth.randomize_module, as the model_* fixtures do.
"""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference'

sys.modules['torchsummary'] = types.SimpleNamespace(summary=None)
sys.path.insert(0, REF)
sys.path.insert(1, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))  # only for gast_b200.synth

import tools.preprocess as _pre                                                      # noqa: E402
import tools.inference as _inf                                                       # noqa: E402
from model.gast_net import SpatioTemporalModel                                       # noqa: E402
from common.skeleton import Skeleton                                                 # noqa: E402
from common.graph_utils import adj_mx_from_skeleton                                  # noqa: E402
from gast_b200 import synth                                                          # noqa: E402
assert _pre.__file__.startswith(REF) and _inf.__file__.startswith(REF), (_pre.__file__, _inf.__file__)

torch.set_grad_enabled(False)
W, H = 1920, 1080
MODEL = dict(J=17, filter_widths=[3, 3, 3], channels=16, seed=41, pad=13)
F32 = np.float32


def model():
    adj = adj_mx_from_skeleton(Skeleton(parents=synth.skeleton_parents(17), joints_left=[], joints_right=[]))
    m = SpatioTemporalModel(adj, 17, 2, 17, MODEL['filter_widths'], channels=MODEL['channels'], dropout=0.05)
    synth.randomize_module(m, MODEL['seed'])
    return m.eval()


def two_person_clip(rs, T=90):
    """two persons, each with all-zero (invalid) frames; their valid frames overlap in part"""
    kp = np.zeros((2, T, 17, 2), F32)
    sc = np.zeros((2, T, 17), F32)
    base = np.array([[700., 400.], [1200., 450.]], F32)
    for p, (lo, hi) in enumerate(((0, 70), (25, T))):
        walk = np.cumsum(rs.standard_normal((T, 1, 2)) * 4, axis=0)
        pose = base[p] + rs.uniform(-120, 120, (1, 17, 2)) + walk + rs.standard_normal((T, 17, 2)) * 3
        kp[p, lo:hi] = pose[lo:hi]
        sc[p, lo:hi] = rs.uniform(0.05, 1.0, (hi - lo, 17))
    kp[0, [3, 40]] = 0                       # holes inside each person's span
    sc[0, [3, 40]] = 0
    kp[1, 60] = 0
    sc[1, 60] = 0
    return kp, sc


def chain(out, name, kp, sc, m):
    """h36m_coco_format -> revise_kpts -> gen_pose -> revise_skes, every stage recorded"""
    out[name + '_kp'], out[name + '_sc'] = kp, sc
    hk, hs, vf = _pre.h36m_coco_format(kp.copy(), sc.copy())
    out[name + '_h36m_kpts'], out[name + '_h36m_scores'] = hk, hs
    out[name + '_n_person'] = np.array(len(vf))
    for p, f in enumerate(vf):
        out['%s_valid%d' % (name, p)] = np.asarray(f, np.int64)
    re = _pre.revise_kpts(hk.copy(), hs.copy(), vf)
    out[name + '_re_kpts'] = re
    pred = _inf.gen_pose(re.copy(), vf, W, H, m, MODEL['pad'], 0)
    for p, q in enumerate(pred):
        out['%s_pose%d' % (name, p)] = np.asarray(q, F32)
    out[name + '_skes'] = _pre.revise_skes([q.copy() for q in pred], re.copy(), vf)


def main():
    out = {}
    m = model()
    rs = np.random.RandomState(71)
    # --- baseball.json: one person plus an empty second slot that h36m_coco_format drops
    kp, sc, label, label_index = _pre.load_json(os.path.join(REF, 'data/keypoints/baseball.json'))
    out['baseball_label'], out['baseball_label_index'] = np.array(label), np.array(label_index)
    chain(out, 'baseball', kp, sc, m)
    # --- a synthetic two-person clip
    chain(out, 'two', *two_person_clip(rs), m)
    # --- revise_kpts: every repair rule, the no-change combinations, scores at float32(0.3) and its neighbours
    T = 80
    rk = rs.uniform(0, 1000, (1, T, 17, 2)).astype(F32)
    rsc = rs.uniform(0.31, 1.0, (1, T, 17)).astype(F32)
    t3 = F32(0.3)
    near = np.array([np.nextafter(t3, F32(0)), t3, np.nextafter(t3, F32(1))], F32)
    for t in range(16):                      # all 16 low/high combinations of joints [2, 3, 5, 6]
        for b, j in enumerate((2, 3, 5, 6)):
            rsc[0, t, j] = 0.1 if (t >> b) & 1 else 0.9
    for t in range(16, T):                   # the threshold itself and one ulp either side
        rsc[0, t, [2, 3, 5, 6]] = near[rs.randint(0, 3, 4)]
    rsc[0, 16, [2, 3, 5, 6]] = near[0]
    rsc[0, 17, [2, 3, 5, 6]] = near[1]
    rsc[0, 18, [2, 3, 5, 6]] = near[2]
    valid = np.array([t for t in range(T) if t not in (7, 33)], np.int64)
    out['rk_kpts'], out['rk_scores'], out['rk_valid'] = rk, rsc, valid
    out['rk_out'] = _pre.revise_kpts(rk.copy(), rsc.copy(), [valid])
    # --- revise_skes on random poses: one person, two persons
    re2 = out['two_re_kpts']
    v2 = [out['two_valid0'], out['two_valid1']]
    for n in (1, 2):
        pred = [rs.standard_normal((len(v2[p]), 17, 3)).astype(F32) for p in range(n)]
        for p in range(n):
            out['skes%d_pred%d' % (n, p)] = pred[p]
        out['skes%d_out' % n] = _pre.revise_skes([q.copy() for q in pred], re2[:n].copy(), v2[:n])
    # --- two persons without a common valid frame
    dis = [np.arange(0, 20, dtype=np.int64), np.arange(20, 40, dtype=np.int64)]
    dk = rs.uniform(0, 1000, (2, 40, 17, 2)).astype(F32)
    dp = [rs.standard_normal((20, 17, 3)).astype(F32) for _ in range(2)]
    try:
        _pre.revise_skes(dp, dk, dis)
        raised = False
    except ValueError:
        raised = True
    assert raised
    out['disjoint_kpts'], out['disjoint_pred0'], out['disjoint_pred1'] = dk, dp[0], dp[1]
    out['disjoint_valid0'], out['disjoint_valid1'] = dis[0], dis[1]
    out['disjoint_raises'] = np.array(raised)
    # --- revise_skes_real_time, M persons of one tick at two image widths
    for M in (1, 2, 64):
        for width in (1920, 1280):
            pred = rs.standard_normal((M, 17, 3)).astype(F32)
            k = rs.uniform(0, width, (M, 17, 2)).astype(F32)
            key = 'rt_M%d_w%d' % (M, width)
            out[key + '_pred'], out[key + '_kpts'] = pred, k
            out[key + '_out'] = _pre.revise_skes_real_time(pred.copy(), k.copy(), width)
    out['meta'] = np.array(json.dumps(dict(numpy=np.__version__, width=W, height=H, gen_pose=MODEL,
                                           rt_M=[1, 2, 64], rt_width=[1920, 1280])))
    np.savez_compressed(os.path.join(HERE, 'preprocess_17.npz'), **out)
    print('preprocess_17', {k: getattr(v, 'shape', None) for k, v in out.items()})


if __name__ == '__main__':
    main()
