"""Golden dataset preparation from the UNMODIFIED reference: common/camera.py world_to_camera and project_to_2d,
main.load_data on small synthetic Human3.6M and HumanEva npz files (extra detection frames to trim), the ground-truth
2D keypoints of data/prepare_data_h36m.py:113-121 loaded back through main.load_data('gt'), and main.fetch with
downsample 1 and 5.

Run where an original checkout is at hand (found as oracle/make_ref.py finds it, or given as the argument):
    python tests/golden/make_golden_dataset.py [<original GAST-Net checkout>]
Writes tests/golden/dataset_camera.npz, dataset_h36m.npz and dataset_humaneva.npz (and nothing else).  The synthetic
inputs come from tests/datasetref.py (synth_h36m, synth_humaneva, seeded); the results are flattened in the
reference's iteration order, with the order listed in 'meta', beside each segment's camera parameters.
"""
import importlib
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.dirname(HERE))
from oracle import make_ref                                                         # noqa: E402
import datasetref as DR                                                             # noqa: E402
REF = make_ref.find_reference(sys.argv[1] if len(sys.argv) > 1 else None)
assert REF, 'no original GAST-Net checkout found'

sys.path.insert(0, REF)
from common.camera import world_to_camera, project_to_2d, image_coordinates        # noqa: E402
from tools.utils import wrap                                                        # noqa: E402
import common.camera as _ref_cam                                                    # noqa: E402
assert _ref_cam.__file__.startswith(REF), _ref_cam.__file__
sys.modules.setdefault('torchsummary', types.SimpleNamespace(summary=None))     # imported by model/, never called
import main as _ref_main                                                            # noqa: E402
assert _ref_main.__file__.startswith(REF), _ref_main.__file__


def camera_cases():
    """world_to_camera on random points with two cameras; project_to_2d with one random camera per row"""
    rs = np.random.RandomState(31)
    out = {}
    for k in range(2):
        X = (rs.standard_normal((600, 17, 3)) * 1.5).astype(np.float32)
        R = rs.standard_normal(4).astype(np.float32)
        R = (R / np.linalg.norm(R)).astype(np.float32)
        t = (rs.standard_normal(3) * 3).astype(np.float32)
        out['w2c%d_X' % k], out['w2c%d_R' % k], out['w2c%d_t' % k] = X, R, t
        out['w2c%d_out' % k] = world_to_camera(X, R=R, t=t)
    N = 64
    X = (rs.standard_normal((N, 40, 3)) * 0.6).astype(np.float32)
    X[..., 2] = np.abs(X[..., 2]) + 3.5
    cam = np.concatenate([rs.uniform(1.9, 2.4, (N, 2)), rs.uniform(-0.05, 0.05, (N, 2)), rs.uniform(-0.25, 0.25, (N, 3)),
                          rs.uniform(-3e-3, 3e-3, (N, 2))], 1).astype(np.float32)
    out['proj_X'], out['proj_cam'] = X, cam
    out['proj_out'] = wrap(project_to_2d, X, cam)
    return out


def flatten(prefix, nested, order):
    """nested[subject][action][cam] arrays -> concatenated array + lengths, in `order` [(subject, action, cam)]"""
    arrs = [np.asarray(nested[s][a][c]) for s, a, c in order]
    return {prefix: np.concatenate(arrs, 0), prefix + '_len': np.array([len(x) for x in arrs], np.int64)}


def flat_list(prefix, lst):
    if lst is None:
        return {prefix + '_none': np.array(1)}
    return {prefix: np.concatenate([np.asarray(x) for x in lst], 0), prefix + '_len': np.array([len(x) for x in lst])}


def run_dataset(name, pos3d, pos2d, keypoints_type, fetch_subjects):
    """write the npz files into data/ of a temporary directory, then the reference's own load_data and fetch"""
    out, meta = {}, {}
    with tempfile.TemporaryDirectory() as d:
        ds_name = 'h36m' if name == 'h36m' else 'humaneva15'
        DR.write_data(d, ds_name, keypoints_type, pos3d, pos2d)
        cwd = os.getcwd()
        os.chdir(d)
        try:
            for mod in ('common.skeleton', 'common.h36m_dataset', 'common.humaneva_dataset'):   # fresh skeletons
                if mod in sys.modules:
                    importlib.reload(sys.modules[mod])
            args = types.SimpleNamespace(dataset=ds_name, keypoints=keypoints_type)
            keypoints, dataset, _, _, _, _, _ = _ref_main.load_data(args)
            if name == 'h36m':                          # the -k gt keypoints, as prepare_data_h36m.py writes them
                gt = {}
                for subject in dataset.subjects():
                    gt[subject] = {}
                    for action in dataset[subject].keys():
                        anim = dataset[subject][action]
                        gt[subject][action] = []
                        for cam in anim['cameras']:
                            p3 = world_to_camera(anim['positions'], R=cam['orientation'], t=cam['translation'])
                            p2 = wrap(project_to_2d, p3, cam['intrinsic'], unsqueeze=True)
                            gt[subject][action].append(image_coordinates(p2, w=cam['res_w'], h=cam['res_h'])
                                                       .astype('float32'))
                np.savez_compressed(os.path.join(d, 'data', 'data_2d_h36m_gt.npz'), positions_2d=gt,
                                    metadata={'layout_name': 'h36m', 'num_joints': 17,
                                              'keypoints_symmetry': [[4, 5, 6, 11, 12, 13], [1, 2, 3, 14, 15, 16]]})
                importlib.reload(sys.modules['common.h36m_dataset'])
                gt_kp, _, _, _, _, _, _ = _ref_main.load_data(types.SimpleNamespace(dataset='h36m', keypoints='gt'))
        finally:
            os.chdir(cwd)
    order3 = [(s, a, c) for s in dataset.subjects() for a in dataset[s].keys()
              for c in range(len(dataset[s][a]['positions_3d']))]
    order2 = [(s, a, c) for s in keypoints for a in keypoints[s] for c in range(len(keypoints[s][a]))]
    out.update(flatten('pos3d', {s: {a: dataset[s][a]['positions_3d'] for a in dataset[s].keys()}
                                 for s in dataset.subjects()}, order3))
    out.update(flatten('kp2d', keypoints, order2))
    cams = dataset.cameras()
    out['seg3_qt'] = np.array([np.concatenate([dataset[s][a]['cameras'][c]['orientation'],
                                               dataset[s][a]['cameras'][c]['translation']]) for s, a, c in order3],
                              np.float32)
    out['seg3_res'] = np.array([(dataset[s][a]['cameras'][c]['res_w'], dataset[s][a]['cameras'][c]['res_h'])
                                for s, a, c in order3], np.int64)
    out['seg2_res'] = np.array([(cams[s][c]['res_w'], cams[s][c]['res_h']) for s, a, c in order2], np.int64)
    if name == 'h36m':
        out['seg3_intr'] = np.array([dataset[s][a]['cameras'][c]['intrinsic'] for s, a, c in order3], np.float32)
        out.update(flatten('gt2d', gt_kp, order3))
    for ds in (1, 5):
        cams, p3, p2 = _ref_main.fetch(fetch_subjects, None, dataset, keypoints, downsample=ds)
        out.update(flat_list('fetch%d_cam' % ds, cams))
        out.update(flat_list('fetch%d_3d' % ds, p3))
        out.update(flat_list('fetch%d_2d' % ds, p2))
    meta['order3'], meta['order2'], meta['fetch_subjects'] = order3, order2, fetch_subjects
    return out, meta


def main():
    np.savez_compressed(os.path.join(HERE, 'dataset_camera.npz'), **camera_cases())
    for name, synth, kt, subjects in (('h36m', DR.synth_h36m, 'cpn_ft_h36m_dbb', ['S9', 'S1']),
                                      ('humaneva', DR.synth_humaneva, 'detectron_pt_coco', ['Train/S1', 'Validate/S2'])):
        pos3d, pos2d = synth()
        out, meta = run_dataset(name, pos3d, pos2d, kt, subjects)
        np.savez_compressed(os.path.join(HERE, 'dataset_%s.npz' % name), meta=json.dumps(meta), **out)
        print(name, {k: v.shape for k, v in out.items() if hasattr(v, 'shape')})


if __name__ == '__main__':
    main()
