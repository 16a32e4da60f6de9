"""Dataset preparation without a GPU: the numpy restatement of the kernels' arithmetic (tests/datasetref.py) against
the unmodified reference's goldens (tests/golden/make_golden_dataset.py) bit for bit, PreparedDataset's fetch and
test_set order against main.fetch and trainval.py's grouping, and prepare's refusals, which come before any upload."""
import numpy as np
import pytest
import torch

import datasetref as DR
from conftest import load_golden
from gast_b200 import dataset as D
from gast_b200.engine import GastError


def _golden(name):
    g = load_golden('dataset_' + name)
    return g, g['meta']


def _inputs(name):
    pos3d, pos2d = (DR.synth_h36m if name == 'h36m' else DR.synth_humaneva)()
    if name == 'h36m':
        pos3d = {s: {a: p[:, DR.H36M_KEPT] for a, p in acts.items()} for s, acts in pos3d.items()}
    return pos3d, pos2d


def test_camera_functions_match_the_reference_bit_for_bit():
    g = load_golden('dataset_camera')
    for k in range(2):
        got = DR.world_to_camera(g['w2c%d_X' % k], g['w2c%d_R' % k], g['w2c%d_t' % k])
        assert np.array_equal(got, g['w2c%d_out' % k])
    assert np.array_equal(DR.project_to_2d(g['proj_X'], g['proj_cam']), g['proj_out'])


def test_fma_emulation_rounds_once():
    # a*b + c = 1024 + 2^-13 + 2^-14 - 2^-46: just below a float32 midpoint, which the double sum rounds onto
    a, b = np.float32(2 ** -7 * (1 + 2 ** -16)), np.float32(2 ** -7 * (1 - 2 ** -16))
    c = np.float32(1024 + 2 ** -13)
    assert (np.float64(a) * np.float64(b) + np.float64(c)).astype(np.float32) == np.float32(1024 + 2 ** -12)
    assert DR.fma32(a, b, c) == np.float32(1024 + 2 ** -13)
    assert DR.fma32(np.float32(3), np.float32(5), np.float32(7)) == np.float32(22)


@pytest.mark.parametrize('name', ['h36m', 'humaneva'])
def test_restated_load_data_matches_the_reference_bit_for_bit(name):
    g, meta = _golden(name)
    pos3d, pos2d = _inputs(name)
    qt = g['seg3_qt']
    want3 = DR.split(g, 'pos3d')
    for i, (s, a, c) in enumerate(meta['order3']):
        assert np.array_equal(DR.world_to_camera(pos3d[s][a], qt[i, :4], qt[i, 4:], root_relative=True), want3[i])
    want2 = DR.split(g, 'kp2d')
    for i, (s, a, c) in enumerate(meta['order2']):
        k = pos2d[s][a][c][:len(want2[i])]
        if name == 'humaneva':
            k = DR.coco_humaneva15(k)
        w, h = (int(v) for v in g['seg2_res'][i])
        assert np.array_equal(DR.normalize_screen(k, w, h), want2[i]), (s, a, c)
    if name == 'h36m':
        wantg = DR.split(g, 'gt2d')
        for i, (s, a, c) in enumerate(meta['order3']):
            p = DR.project_to_2d(DR.world_to_camera(pos3d[s][a], qt[i, :4], qt[i, 4:])[None], g['seg3_intr'][i:i + 1])[0]
            w, h = (int(v) for v in g['seg3_res'][i])
            assert np.array_equal(DR.normalize_screen(p, w, h, from_image=True), wantg[i])


def _prepared_from_golden(name):
    """a PreparedDataset of CPU tensors holding the golden's load_data results (fetch and test_set are host logic)"""
    g, meta = _golden(name)
    pos3d, kp2d = DR.split(g, 'pos3d'), DR.split(g, 'kp2d')
    p3, k2, intr, actions = {}, {}, {}, {}
    for i, (s, a, c) in enumerate(meta['order3']):
        p3.setdefault(s, {}).setdefault(a, []).append(torch.from_numpy(pos3d[i]))
        actions.setdefault(s, [])
        if a not in actions[s]:
            actions[s].append(a)
        if 'seg3_intr' in g:
            row = intr.setdefault(s, [])
            if len(row) <= c:
                row.append(torch.from_numpy(g['seg3_intr'][i]))
    for i, (s, a, c) in enumerate(meta['order2']):
        k2.setdefault(s, {}).setdefault(a, []).append(torch.from_numpy(kp2d[i]))
        if 'seg3_intr' not in g:
            intr.setdefault(s, [None] * 3)
    return D.PreparedDataset(p3, k2, intr, actions), g, meta


@pytest.mark.parametrize('name', ['h36m', 'humaneva'])
@pytest.mark.parametrize('downsample', [1, 5])
def test_fetch_order_matches_main_fetch(name, downsample):
    ds, g, meta = _prepared_from_golden(name)
    cams, p3, p2 = ds.fetch(meta['fetch_subjects'], None, downsample)
    assert [np.asarray(p) for p in p2] and all(np.array_equal(a.numpy(), b)
                                               for a, b in zip(p2, DR.split(g, 'fetch%d_2d' % downsample)))
    assert len(p2) == len(g['fetch%d_2d_len' % downsample])
    want3 = DR.split(g, 'fetch%d_3d' % downsample)
    assert len(p3) == len(want3) and all(np.array_equal(a.numpy(), b) for a, b in zip(p3, want3))
    if 'fetch%d_cam_none' % downsample in g:
        assert cams is None
    else:
        wantc = DR.split(g, 'fetch%d_cam' % downsample)
        assert len(cams) == len(wantc) and all(np.array_equal(a.numpy(), b) for a, b in zip(cams, wantc))


def test_test_set_groups_like_run_evaluation():
    ds, g, meta = _prepared_from_golden('h36m')
    p3, p2, groups = ds.test_set(['S9', 'S1'])
    # all_actions: action names in first-seen order over the subjects, each group's (subject, action) pairs in order
    want = [('Directions', 'S9', 'Directions'), ('Walking', 'S9', 'Walking'), ('Walking', 'S1', 'Walking'),
            ('Walking', 'S1', 'Walking 1'), ('Eating', 'S1', 'Eating 2')]
    assert groups == [w[0] for w in want for _ in range(4)]
    got = [p for p in p3]
    exp = [ds.positions_3d[s][a][c] for _, s, a in want for c in range(4)]
    assert all(x is y or torch.equal(x, y) for x, y in zip(got, exp)) and len(got) == len(exp)
    _, _, gs = ds.test_set(['S9', 'S1'], by_subject=True)
    assert gs == [k for k in [('S9', 'Directions'), ('S9', 'Walking'), ('S1', 'Walking'), ('S1', 'Eating')]
                  for _ in range(4 * (2 if k == ('S1', 'Walking') else 1))]
    _, p2f, gf = ds.test_set(['S9', 'S1'], action_filter=['Walk'], downsample=5)
    assert set(gf) == {'Walking'} and len(gf) == 12 and p2f[0].shape[0] == (19 + 4) // 5


def _h36m_standin():
    pos3d, pos2d = _inputs('h36m')
    q = np.array([0.5, -0.5, 0.5, -0.5], np.float32)
    cam = {'orientation': q, 'translation': np.zeros(3, np.float32), 'res_w': 1000, 'res_h': 1002,
           'intrinsic': np.ones(9, np.float32)}
    return pos3d, pos2d, {s: [dict(cam) for _ in range(4)] for s in pos3d}


def test_prepare_refuses_what_load_data_asserts_before_any_upload():
    pos3d, pos2d, cams = _h36m_standin()

    def refused(p3, p2, match, humaneva=False):
        with pytest.raises(GastError, match=match):
            D.prepare(DR.MocapStandIn(p3, cams), p2, humaneva=humaneva)

    refused(pos3d, {s: v for s, v in pos2d.items() if s != 'S9'}, 'subject S9 is missing')
    p2 = {s: dict(v) for s, v in pos2d.items()}
    del p2['S1']['Walking 1']
    refused(pos3d, p2, 'action Walking 1 of subject S1 is missing')
    p2 = {s: {a: list(c) for a, c in v.items()} for s, v in pos2d.items()}
    p2['S1']['Eating 2'][2] = p2['S1']['Eating 2'][2][:10]
    refused(pos3d, p2, 'camera 2 has 10 detected frames for 23 mocap frames')
    p2 = {s: {a: list(c) for a, c in v.items()} for s, v in pos2d.items()}
    p2['S9']['Walking'] = p2['S9']['Walking'][:3]
    refused(pos3d, p2, '3 detection cameras and 4 mocap cameras')
    p3 = {s: dict(v) for s, v in pos3d.items()}
    p3['S1']['Walking'] = p3['S1']['Walking'].astype(np.float64)
    refused(p3, pos2d, 'positions of S1 Walking must be a float32')
    p2 = {s: {a: [k[:, :15] for k in c] for a, c in v.items()} for s, v in pos2d.items()}
    refused(pos3d, p2, r'HumanEva detections must be \(T, 17, 2\)', humaneva=True)
    p2 = {s: {a: list(c) for a, c in v.items()} for s, v in pos2d.items()}
    p2['S1']['Walking'][0] = p2['S1']['Walking'][0][..., :1]
    refused(pos3d, p2, 'detections of S1 Walking must be')
    cams['S1'][1] = {'res_w': 1000, 'res_h': 1000}
    refused(pos3d, pos2d, 'camera 1 of S1 has no extrinsics')


def test_fetch_refuses_subset():
    ds, _, meta = _prepared_from_golden('h36m')
    with pytest.raises(GastError, match='subset < 1'):
        ds.fetch(['S1'], subset=0.5)
    with pytest.raises(GastError, match='subject S7 is not in the keypoints'):
        ds.fetch(['S7'])
