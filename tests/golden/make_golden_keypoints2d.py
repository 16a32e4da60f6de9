"""Golden outputs of the 2D pose net's crop and heatmap decode from the UNMODIFIED reference
(lib/pose/hrnet/lib/utils/utilitys.py: box_to_center_scale, PreProcess; lib/pose/hrnet/lib/utils/transforms.py:
get_affine_transform; lib/pose/hrnet/lib/utils/inference.py: get_final_preds), with cv2 4.13 and torchvision 0.26.

Run in the build container only (the GPU box has no reference checkout and may have no cv2):
    python tests/golden/make_golden_keypoints2d.py
Writes tests/golden/keypoints2d.npz (and nothing else).  Frames and heatmaps are not stored: they are made by the
integer formulas of tests/keypoints2dref.py (synth_frames, synth_heatmaps, edge_case_heatmaps).  The config is a
SimpleNamespace (yacs is not needed).
"""
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference'
HRNET = os.path.join(REF, 'lib', 'pose', 'hrnet')

sys.path.insert(0, os.path.join(HRNET, 'lib'))
sys.path.insert(1, os.path.join(HRNET, 'pose_estimation'))        # utilitys.py imports _init_paths
sys.path.insert(2, os.path.join(REPO, 'tests'))

import cv2                                                          # noqa: E402
from utils import utilitys as _U                                    # noqa: E402
from utils import transforms as _T                                  # noqa: E402
from utils import inference as _I                                   # noqa: E402
import keypoints2dref as R                                          # noqa: E402
assert all(m.__file__.startswith(REF) for m in (_U, _T, _I)), (_U.__file__, _T.__file__, _I.__file__)

F, H, W = 3, 1080, 1920
SMALL = (48, 64)                    # every box's warp at a small crop size
FULL = (288, 384)                  # w48_384x288's crop, stored for the first FULL_N boxes
FULL_N = 1
PRE_SIZE = (48, 64)                # PreProcess's float crops
HEATMAPS = [(72, 96), (48, 64)]    # (hw, hh)


def boxes():
    """(16, 4) float64 on a 0.01 grid, as gen_video_kpts rounds them, with their frames: people-shaped boxes inside
    the frame, partly outside on every side, wide, tall, tiny and one covering more than the frame"""
    rs = np.random.default_rng(7)
    out = []
    for k in range(10):
        w, h = rs.uniform(80, 420), rs.uniform(200, 900)
        x1, y1 = rs.uniform(0, W - w), rs.uniform(0, H - h)
        out.append([x1, y1, x1 + w, y1 + h])
    out += [[-120.37, 300.5, 180.21, 900.77], [1700.11, -80.4, 2050.9, 500.33], [400.0, 800.25, 760.5, 1300.12],
            [10.0, 10.0, 1500.0, 200.0], [900.0, 100.0, 920.0, 1000.0], [-300.0, -200.0, 2200.0, 1300.0]]
    b = np.array([[round(v, 2) for v in list(np.asarray(r, np.float64))] for r in out])
    return b, np.arange(len(b)) % F


def main():
    frames = R.synth_frames(F, H, W)
    bx, bf = boxes()
    n = len(bx)
    centers, scales, fwd_small, fwd_full = [], [], [], []
    inv = {s: [] for s in HEATMAPS}
    warps_small, warps_full = [], []
    for k in range(n):
        box = [v for v in bx[k]]
        c, s = _U.box_to_center_scale(box, H, W)                  # PreProcess's argument order
        centers.append(c)
        scales.append(s)
        ms = _T.get_affine_transform(c, s, 0, list(SMALL))
        mf = _T.get_affine_transform(c, s, 0, list(FULL))
        fwd_small.append(ms)
        fwd_full.append(mf)
        for hs in HEATMAPS:
            inv[hs].append(_T.get_affine_transform(c, s, 0, list(hs), inv=1))
        warps_small.append(cv2.warpAffine(frames[bf[k]], ms, SMALL, flags=cv2.INTER_LINEAR))
        if k < FULL_N:
            warps_full.append(cv2.warpAffine(frames[bf[k]], mf, FULL, flags=cv2.INTER_LINEAR))
    centers, scales = np.stack(centers), np.stack(scales)

    # PreProcess calls: (frame, first box, number of boxes, num_pos)
    cfg = SimpleNamespace(MODEL=SimpleNamespace(IMAGE_SIZE=list(PRE_SIZE)), TEST=SimpleNamespace(POST_PROCESS=True))
    pre_calls = [(0, 0, 2, 2), (1, 2, 1, 2), (2, 3, 3, 2)]
    pre_inputs, pre_centers, pre_scales, pre_fwd = [], [], [], []
    for f, b0, nb, num_pos in pre_calls:
        bb = [list(r) for r in bx[b0:b0 + nb]]
        inputs, img, c, s = _U.PreProcess(frames[f], bb, cfg, num_pos)
        pre_fwd.append(np.stack([_T.get_affine_transform(ci, si, 0, list(PRE_SIZE)) for ci, si in zip(c, s)]))
        pre_inputs.append(inputs.numpy())
        pre_centers.append(np.stack(c))
        pre_scales.append(np.stack(s))

    # get_final_preds on the edge-case maps and smooth maps, records paired with boxes 0..7
    dec = {}
    for hw, hh in HEATMAPS:
        hm = np.concatenate([R.edge_case_heatmaps(hh, hw), R.synth_heatmaps(4, 17, hh, hw, seed=3)])
        m = hm.shape[0]
        for post in (True, False):
            cfgp = SimpleNamespace(TEST=SimpleNamespace(POST_PROCESS=post))
            with np.errstate(invalid='ignore'):
                p, mv = _I.get_final_preds(cfgp, hm.copy(), centers[:m], scales[:m])
            key = 'dec_%dx%d_%s' % (hw, hh, 'post' if post else 'plain')
            dec[key + '_preds'] = p.astype(np.float32)
            dec[key + '_maxvals'] = mv

    meta = dict(F=F, H=H, W=W, small=SMALL, full=FULL, full_n=FULL_N, pre_size=PRE_SIZE, pre_calls=pre_calls,
                heatmaps=HEATMAPS, cv2=cv2.__version__, torch=torch.__version__, numpy=np.__version__)
    out = dict(boxes=bx, box_frame=bf.astype(np.int64), centers=centers, scales=scales,
               fwd_small=np.stack(fwd_small), fwd_full=np.stack(fwd_full),
               warps_small=np.stack(warps_small), warps_full=np.stack(warps_full),
               meta=np.array(json.dumps(meta)), **dec)
    for hw, hh in HEATMAPS:
        out['inv_%dx%d' % (hw, hh)] = np.stack(inv[(hw, hh)])
    for i, (x, c, s, m) in enumerate(zip(pre_inputs, pre_centers, pre_scales, pre_fwd)):
        out['pre%d_inputs' % i], out['pre%d_centers' % i], out['pre%d_scales' % i] = x, c, s
        out['pre%d_fwd' % i] = m
    path = os.path.join(HERE, 'keypoints2d.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
