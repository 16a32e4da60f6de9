"""GPU: preparing a synthetic Human3.6M-sized dataset, the reference's host way against gast_b200.dataset.

The dataset: `--actions` actions spread over the seven Human3.6M subjects, `--frames` mocap frames each (32 joints,
seeded), four cameras of 17-joint detections with up to 5 extra frames each, written uncompressed into a temporary
data/ directory.  Two ways to prepare it, alternated `--reps` times in one process:
  * reference: the staged, unchanged main.load_data + main.fetch of the training and the test subjects
    (oracle/_ref/main.py), and the ground-truth 2D keypoints as data/prepare_data_h36m.py:113-121 computes them,
    normalised as main.load_data normalises the `gt` keypoints;
  * device: the same Human36mDataset construction and detection load, then gast_b200.dataset.prepare, the two fetch
    calls and ground_truth_2d, ending in a device synchronise.
Both sides read the same npz files; the read alone (Human36mDataset + np.load of the detections) is timed too.
Prints one JSON line per run (host clock), the first with the card's name and power limit read in the same run.
Needs oracle/_ref/ (build() stages it).

    python tools/dataset_bench.py [--actions 210] [--frames 4300] [--reps 3]
"""
import argparse
import contextlib
import importlib
import io
import json
import os
import sys
import tempfile
import time
import types

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, 'gast-net-3dposeestimation_b200')
REF = os.path.join(REPO, 'oracle', '_ref')
sys.path[:0] = [PKG, REPO, os.path.dirname(os.path.abspath(__file__))]
from gast_b200 import dataset as D  # noqa: E402
from eval_bench import card  # noqa: E402

SUBJECTS = ['S1', 'S5', 'S6', 'S7', 'S8', 'S9', 'S11']
TRAIN, TEST = ['S1', 'S5', 'S6', 'S7', 'S8'], ['S9', 'S11']


def write(root, n_actions, frames, seed=0):
    rs = np.random.RandomState(seed)
    pos3d, pos2d = {s: {} for s in SUBJECTS}, {s: {} for s in SUBJECTS}
    for i in range(n_actions):
        s, a = SUBJECTS[i % len(SUBJECTS)], 'Action%d %d' % (i // len(SUBJECTS), i % 2)
        root_t = rs.uniform(-1, 1, (1, 1, 3)).astype(np.float32) * [1, 1, 0] + np.float32([0, 0, 0.9])
        pos3d[s][a] = (root_t + 0.4 * rs.standard_normal((frames, 32, 3))).astype(np.float32)
        pos2d[s][a] = [rs.uniform(0, 1000, (frames + int(rs.randint(0, 6)), 17, 2)).astype(np.float32) for _ in range(4)]
    os.makedirs(os.path.join(root, 'data'))
    np.savez(os.path.join(root, 'data', 'data_3d_h36m.npz'), positions_3d=pos3d)
    np.savez(os.path.join(root, 'data', 'data_2d_h36m_cpn_ft_h36m_dbb.npz'), positions_2d=pos2d,
             metadata={'layout_name': 'coco', 'num_joints': 17,
                       'keypoints_symmetry': [[1, 3, 5, 7, 9, 11, 13, 15], [2, 4, 6, 8, 10, 12, 14, 16]]})


def read():
    """Human36mDataset and the detections, as main.load_data reads them"""
    importlib.reload(sys.modules['common.h36m_dataset'])     # a fresh module-level skeleton per construction
    from common.h36m_dataset import Human36mDataset
    ds = Human36mDataset('data/data_3d_h36m.npz', 'cpn_ft_h36m_dbb')
    kp = np.load('data/data_2d_h36m_cpn_ft_h36m_dbb.npz', allow_pickle=True)['positions_2d'].item()
    return ds, kp


def run_reference(main, cam):
    t0 = time.perf_counter()
    importlib.reload(sys.modules['common.h36m_dataset'])
    keypoints, dataset, _, _, _, _, _ = main.load_data(types.SimpleNamespace(dataset='h36m', keypoints='cpn_ft_h36m_dbb'))
    main.fetch(TRAIN, None, dataset, keypoints, downsample=1)
    main.fetch(TEST, None, dataset, keypoints, downsample=1)
    t1 = time.perf_counter()
    n = 0
    for subject in dataset.subjects():                        # prepare_data_h36m.py:113-121, then main.py:101
        for action in dataset[subject].keys():
            anim = dataset[subject][action]
            for c in anim['cameras']:
                p3 = cam.world_to_camera(anim['positions'], R=c['orientation'], t=c['translation'])
                p2 = cam.wrap(cam.project_to_2d, p3, c['intrinsic'], unsqueeze=True)
                k = cam.image_coordinates(p2, w=c['res_w'], h=c['res_h']).astype('float32')
                k[..., :2] = cam.normalize_screen_coordinates(k[..., :2], w=c['res_w'], h=c['res_h'])
                n += k.shape[0]
    return t1 - t0, time.perf_counter() - t0, n


def run_device():
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ds, kp = read()
    t_read = time.perf_counter() - t0
    prep = D.prepare(ds, kp)
    prep.fetch(TRAIN, None, 1)
    prep.fetch(TEST, None, 1)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    prep.ground_truth_2d()
    torch.cuda.synchronize()
    return t_read, t1 - t0, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--actions', type=int, default=210)
    ap.add_argument('--frames', type=int, default=4300)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    print(json.dumps({'card': card(), 'torch_threads': torch.get_num_threads()}), flush=True)
    if not os.path.exists(os.path.join(REF, 'main.py')):
        raise SystemExit('oracle/_ref/ is not staged (python oracle/make_ref.py <original checkout>)')
    sys.path[:] = [PKG, REF] + [p for p in sys.path if p not in (PKG, REF)]
    with tempfile.TemporaryDirectory() as d:
        write(d, args.actions, args.frames)
        os.chdir(d)
        import main                                           # oracle/_ref/main.py, unchanged
        import common.camera as cam                           # oracle/_ref/common/camera.py
        import common.h36m_dataset  # noqa: F401
        print(json.dumps({'actions': args.actions, 'frames': args.frames, 'cameras': 4,
                          'bytes': sum(os.path.getsize(os.path.join(d, 'data', f)) for f in os.listdir('data'))}),
              flush=True)
        with contextlib.redirect_stdout(io.StringIO()):
            run_device()                                      # warm-up: modules, allocator
        for rep in range(args.reps):
            out = {'rep': rep}
            with contextlib.redirect_stdout(io.StringIO()):
                out['reference_load_fetch_s'], out['reference_with_gt_s'], out['gt_frames'] = run_reference(main, cam)
                out['read_s'], out['device_load_fetch_s'], out['device_with_gt_s'] = run_device()
            out['speedup_load_fetch'] = out['reference_load_fetch_s'] / out['device_load_fetch_s']
            out['speedup_with_gt'] = out['reference_with_gt_s'] / out['device_with_gt_s']
            print(json.dumps(out), flush=True)
        os.chdir(REPO)


if __name__ == '__main__':
    main()
