"""Mocap datasets prepared on the device (gast_b200.dataset, the dataset kernels of csrc/pipeline.cuh):
  * every kernel equals the unmodified reference's goldens bit for bit (tests/golden/make_golden_dataset.py);
  * a segmented launch equals one call per sequence bit for bit;
  * project_to_2d's backward is within 1e-6 relative of fp64 autograd of the projection formula;
  * prepare + fetch equal the unchanged main.load_data + main.fetch (oracle/_ref/) bit for bit;
  * EpochTrainer epochs and evaluate_sequences scores fed from the device-prepared splits equal those fed from the
    reference's host-prepared ones bit for bit;
  * prepare, fetch, test_set and ground_truth_2d make no host synchronisation."""
import importlib
import sys

import numpy as np
import pytest
import torch

import datasetref as DR
from conftest import load_golden
from gast_b200 import dataset as D
from gast_b200 import pipeline as P
from gast_b200 import synth
from test_unchanged_callers import LEFT, RIGHT, callers, needs_callers  # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu


def _golden(name):
    g = load_golden('dataset_' + name)
    return g, g['meta']


def _standin(name):
    """the golden's synthetic dataset behind MocapDataset's interface, with the cameras main.load_data used, and the
    raw positions_2d dict"""
    g, meta = _golden(name)
    pos3d, pos2d = (DR.synth_h36m if name == 'h36m' else DR.synth_humaneva)()
    if name == 'h36m':
        pos3d = {s: {a: p[:, DR.H36M_KEPT] for a, p in acts.items()} for s, acts in pos3d.items()}
    cams = {}
    for i, (s, a, c) in enumerate(meta['order3']):
        row = cams.setdefault(s, [])
        if len(row) <= c:
            cam = {'orientation': g['seg3_qt'][i, :4], 'translation': g['seg3_qt'][i, 4:],
                   'res_w': int(g['seg3_res'][i, 0]), 'res_h': int(g['seg3_res'][i, 1])}
            if 'seg3_intr' in g:
                cam['intrinsic'] = g['seg3_intr'][i]
            row.append(cam)
    return DR.MocapStandIn(pos3d, cams), pos2d, g, meta


def _eq(got, want):
    got = got.cpu().numpy() if isinstance(got, torch.Tensor) else np.asarray(got)
    return got.shape == np.shape(want) and np.array_equal(got, want)


def test_camera_kernels_equal_the_reference_goldens():
    from device.common.camera import world_to_camera, project_to_2d
    g = load_golden('dataset_camera')
    for k in range(2):
        x = torch.from_numpy(g['w2c%d_X' % k]).cuda()
        assert _eq(world_to_camera(x, g['w2c%d_R' % k], g['w2c%d_t' % k]), g['w2c%d_out' % k])
        assert np.array_equal(world_to_camera(g['w2c%d_X' % k], g['w2c%d_R' % k], g['w2c%d_t' % k]), g['w2c%d_out' % k])
    assert _eq(project_to_2d(torch.from_numpy(g['proj_X']).cuda(), torch.from_numpy(g['proj_cam']).cuda()), g['proj_out'])
    assert np.array_equal(project_to_2d(g['proj_X'], g['proj_cam']), g['proj_out'])


@pytest.mark.parametrize('name', ['h36m', 'humaneva'])
def test_prepare_fetch_and_ground_truth_equal_the_goldens(name):
    ds_in, pos2d, g, meta = _standin(name)
    ds = D.prepare(ds_in, pos2d, humaneva=name == 'humaneva')
    for (s, a, c), want in zip(meta['order3'], DR.split(g, 'pos3d')):
        assert _eq(ds.positions_3d[s][a][c], want), (s, a, c)
    for (s, a, c), want in zip(meta['order2'], DR.split(g, 'kp2d')):
        assert _eq(ds.keypoints[s][a][c], want), (s, a, c)
    for k in (1, 5):
        cams, p3, p2 = ds.fetch(meta['fetch_subjects'], None, k)
        assert len(p2) == len(g['fetch%d_2d_len' % k])
        assert all(_eq(x, y) for x, y in zip(p2, DR.split(g, 'fetch%d_2d' % k)))
        assert len(p3) == len(g['fetch%d_3d_len' % k])
        assert all(_eq(x, y) for x, y in zip(p3, DR.split(g, 'fetch%d_3d' % k)))
        if name == 'h36m':
            assert all(_eq(x, y) for x, y in zip(cams, DR.split(g, 'fetch%d_cam' % k)))
        else:
            assert cams is None
    if name == 'h36m':
        gt = ds.ground_truth_2d()
        for (s, a, c), want in zip(meta['order3'], DR.split(g, 'gt2d')):
            assert _eq(gt.keypoints[s][a][c], want), (s, a, c)
        assert gt.positions_3d is ds.positions_3d
    else:
        with pytest.raises(P.GastError, match='needs intrinsics'):
            ds.ground_truth_2d()


def test_humaneva_remap_is_a_keypoints_convert_mode():
    rs = np.random.RandomState(2)
    k = rs.uniform(0, 640, (333, 17, 2)).astype(np.float32)
    out, valid = P.keypoints_convert(torch.from_numpy(k).cuda(), P.KPT_COCO_HUMANEVA)
    assert _eq(out, DR.coco_humaneva15(k)) and bool((valid == 1).all())
    with pytest.raises(P.GastError, match='does not take 16 joints'):
        P.keypoints_convert(torch.from_numpy(k[:, :16]).cuda(), P.KPT_COCO_HUMANEVA)


def _segments(rs, lengths, ncam):
    """sequences x cameras: src (S,), dst (S+1,) frame offsets"""
    starts = np.concatenate([[0], np.cumsum(lengths)])
    src = np.repeat(starts[:-1], ncam).astype(np.int64)
    dst = np.concatenate([[0], np.cumsum(np.repeat(lengths, ncam))]).astype(np.int64)
    return src, dst


def test_segmented_launches_equal_per_sequence_calls():
    from device.common.camera import world_to_camera, project_to_2d
    rs = np.random.RandomState(5)
    lengths, ncam, J = [57, 1, 300, 129], 4, 17
    x = torch.from_numpy((rs.standard_normal((sum(lengths), J, 3)) * 1.3).astype(np.float32)).cuda()
    src, dst = _segments(rs, lengths, ncam)
    S = len(src)
    q = rs.standard_normal((S, 4)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    qt = np.concatenate([q, rs.standard_normal((S, 3)).astype(np.float32) * 4 + [0, 0, 8]], 1).astype(np.float32)
    intr = np.concatenate([rs.uniform(1.9, 2.4, (S, 2)), rs.uniform(-0.05, 0.05, (S, 2)), rs.uniform(-0.25, 0.25, (S, 3)),
                           rs.uniform(-3e-3, 3e-3, (S, 2))], 1).astype(np.float32)
    res = [(1000, 1002), (1000, 1000), (640, 480), (1920, 1080)] * len(lengths)
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()      # noqa: E731
    n = int(dst[-1])
    cam = P.world_to_camera_segments(x, cu(src), cu(dst), cu(qt), n)
    rel = P.world_to_camera_segments(x, cu(src), cu(dst), cu(qt), n, root_relative=True)
    px = P.project_to_2d_segments(cam.reshape(-1, 3), cu(dst * J), cu(intr))
    wh = cu(np.array([(w, h / w) for w, h in res], np.float64))
    nk = P.normalize_screen_segments(px.reshape(n, J, 2), cu(dst[:-1]), cu(dst), wh, n)
    rt = P.normalize_screen_segments(px.reshape(n, J, 2), cu(dst[:-1]), cu(dst), wh, n, from_image=True)
    for s in range(S):
        T, a, b = lengths[s // ncam], int(dst[s]), int(dst[s + 1])
        xs = x[src[s]:src[s] + T]
        one = world_to_camera(xs, qt[s, :4], qt[s, 4:])
        assert torch.equal(cam[a:b], one)
        assert torch.equal(rel[a:b, 1:], one[:, 1:] - one[:, :1]) and torch.equal(rel[a:b, 0], one[:, 0])
        assert torch.equal(px.reshape(n, J, 2)[a:b], project_to_2d(one, cu(np.tile(intr[s], (T, 1)))))
        w, h = res[s]
        assert torch.equal(nk[a:b], P.normalize_screen(px.reshape(n, J, 2)[a:b], w, h))
        img = P.normalize_screen(px.reshape(n, J, 2)[a:b], w, h, inverse=True)
        assert torch.equal(rt[a:b], P.normalize_screen(img, w, h))
    # extra channels are copied; the trimmed tail of a source is skipped
    k3 = torch.from_numpy(rs.uniform(0, 1000, (40, J, 3)).astype(np.float32)).cuda()
    out = P.normalize_screen_segments(k3, cu(np.array([0, 20])), cu(np.array([0, 15, 25])),
                                      cu(np.array([(1000, 1.002), (640, 0.75)])), 25)
    assert torch.equal(out[:15, :, 2], k3[:15, :, 2]) and torch.equal(out[15:, :, 2], k3[20:30, :, 2])
    assert torch.equal(out[15:, :, :2], P.normalize_screen(k3[20:30, :, :2].contiguous(), 640, 480))


def _project64(X, cam):
    """the Human3.6M projection model (radial k1..k3, tangential p1, p2) in the input's precision"""
    k = cam.reshape(cam.shape[0], 1, 9)
    xy = X[..., :2] / X[..., 2:]
    r2 = (xy ** 2).sum(-1, keepdim=True)
    radial = 1 + k[..., 4:5] * r2 + k[..., 5:6] * r2 ** 2 + k[..., 6:7] * r2 ** 3
    tan = (k[..., 7:9] * xy).sum(-1, keepdim=True)
    return k[..., 0:2] * (xy * (radial + tan) + k[..., 7:9] * r2) + k[..., 2:4]


def test_project_to_2d_backward_against_fp64_autograd():
    from device.common.camera import project_to_2d
    rs = np.random.RandomState(7)
    N = 24
    X = (rs.standard_normal((N, 300, 3)) * 0.7).astype(np.float32)
    X[..., 2] = np.abs(X[..., 2]) + rs.uniform(1.5, 6, (N, 1))
    cam = np.concatenate([rs.uniform(1.9, 2.4, (N, 2)), rs.uniform(-0.05, 0.05, (N, 2)), rs.uniform(-0.25, 0.25, (N, 3)),
                          rs.uniform(-3e-3, 3e-3, (N, 2))], 1).astype(np.float32)
    g = rs.standard_normal((N, 300, 2)).astype(np.float32)
    x = torch.from_numpy(X).cuda().requires_grad_()
    y = project_to_2d(x, torch.from_numpy(cam).cuda())
    (gx,) = torch.autograd.grad(y, x, torch.from_numpy(g).cuda())
    x64 = torch.from_numpy(X).double().requires_grad_()
    (ref,) = torch.autograd.grad(_project64(x64, torch.from_numpy(cam).double()), x64, torch.from_numpy(g).double())
    ref = ref.numpy()
    err = np.abs(gx.cpu().numpy().astype(np.float64) - ref)
    assert (err <= 1e-6 * np.abs(ref) + 1e-12).all(), float((err / (np.abs(ref) + 1e-30)).max())
    with pytest.raises(P.GastError, match='no gradient with respect to the intrinsics'):
        project_to_2d(x, torch.from_numpy(cam).cuda().requires_grad_())


def test_prepare_fetch_and_test_set_make_no_host_sync():
    ds_in, pos2d, g, meta = _standin('h36m')
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        ds = D.prepare(ds_in, pos2d)
        ds.fetch(['S1'], ['Walk'], 5)
        ds.test_set(['S9', 'S1'], by_subject=True)
        gt = ds.ground_truth_2d()
        gt.fetch(['S9'], None, 1)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert _eq(ds.keypoints['S9']['Walking'][3], DR.split(g, 'kp2d')[meta['order2'].index(['S9', 'Walking', 3])])


def _reload_datasets():
    for mod in ('common.h36m_dataset', 'common.humaneva_dataset'):       # fresh module-level skeletons
        if mod in sys.modules:
            importlib.reload(sys.modules[mod])


@needs_callers
@pytest.mark.parametrize('name', ['h36m', 'humaneva'])
def test_prepare_and_fetch_equal_the_unchanged_load_data_and_fetch(callers, name, tmp_path, monkeypatch):
    """the reference's own main.load_data / main.fetch over npz files in a temporary data/ directory.  torch's CPU
    cross product rounds each component as fma(a1, b2, -(a2*b1)) (measured where the goldens were made); the
    committed goldens hold that bit-exact bar independently of this machine's CPU build."""
    import types
    _, mn = callers
    pos3d, pos2d = (DR.synth_h36m if name == 'h36m' else DR.synth_humaneva)(seed=11)
    ds_name, kt = ('h36m', 'cpn_ft_h36m_dbb') if name == 'h36m' else ('humaneva15', 'detectron_pt_coco')
    DR.write_data(str(tmp_path), ds_name, kt, pos3d, pos2d)
    monkeypatch.chdir(tmp_path)
    _reload_datasets()
    keypoints, dataset, _, _, _, _, _ = mn.load_data(types.SimpleNamespace(dataset=ds_name, keypoints=kt))
    raw = np.load('data/data_2d_%s_%s.npz' % (ds_name, kt), allow_pickle=True)['positions_2d'].item()
    ds = D.prepare(dataset, raw, humaneva=name == 'humaneva')
    for s in dataset.subjects():
        for a in dataset[s].keys():
            for c, want in enumerate(dataset[s][a]['positions_3d']):
                assert _eq(ds.positions_3d[s][a][c], want), (s, a, c)
    for s in keypoints:
        for a in keypoints[s]:
            assert len(ds.keypoints[s][a]) == len(keypoints[s][a])
            for c, want in enumerate(keypoints[s][a]):
                assert _eq(ds.keypoints[s][a][c], want), (s, a, c)
    subjects = list(dataset.subjects())[::-1]
    for k, flt in ((1, None), (5, None), (5, ['Walk'])):
        want = mn.fetch(subjects, flt, dataset, keypoints, downsample=k)
        got = ds.fetch(subjects, flt, k)
        for w, x in zip(want, got):
            assert (w is None) == (x is None)
            if w is not None:
                assert len(w) == len(x) and all(_eq(b, a) for a, b in zip(w, x))


def _model(kind, seed=4):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(17), LEFT, RIGHT))
    cls = SpatioTemporalModelOptimized1f if kind == 'o1f' else SpatioTemporalModel
    m = cls(adj, 17, 2, 17, [3, 3, 3], dropout=0.0, channels=32)
    synth.randomize_module(m, seed)
    return m.cuda()


def test_training_and_evaluation_from_device_splits_equal_host_splits():
    """the same epoch and the same scores whether the splits come from prepare + fetch or from the reference's
    host-prepared lists (the goldens hold main.load_data + main.fetch's arrays)"""
    from device.common.generators import ChunkedGenerator
    from gast_b200.evaluation import evaluate_sequences
    from gast_b200.training import EpochTrainer
    ds_in, pos2d, g, meta = _standin('h36m')
    ds = D.prepare(ds_in, pos2d)
    dev_split = ds.fetch(meta['fetch_subjects'], None, 1)
    host_split = (list(g['fetch1_cam'].reshape(-1, 9)), DR.split(g, 'fetch1_3d'), DR.split(g, 'fetch1_2d'))
    results = []
    for cams, p3, p2 in (dev_split, host_split):
        m = _model('o1f').train()
        opt = P.FusedAdam(m.parameters(), lr=1e-3, amsgrad=True)
        gen = ChunkedGenerator(40, cams, p3, p2, 1, pad=13, causal_shift=0, shuffle=True, random_seed=1234,
                               augment=True, kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
        tr = EpochTrainer(m, gen, opt)
        losses = [tr.train_epoch() for _ in range(2)]
        results.append((losses, {k: v.detach().cpu().clone() for k, v in m.state_dict().items()},
                        gen.seqs.cameras.cpu()))
    (l_d, sd_d, c_d), (l_h, sd_h, c_h) = results
    assert l_d == l_h and torch.equal(c_d, c_h)
    assert all(torch.equal(sd_d[k], sd_h[k]) for k in sd_d)

    p3, p2, groups = ds.test_set(['S9', 'S1'])
    order = {tuple(k): i for i, k in enumerate(meta['order3'])}
    h3, h2 = DR.split(g, 'pos3d'), DR.split(g, 'kp2d')
    o2 = {tuple(k): i for i, k in enumerate(meta['order2'])}
    keys = [(s, a, c) for s in ('S9', 'S1') for a in ds._actions[s] for c in range(4)]
    names = [a.split(' ')[0] for _, a, _ in keys]
    first = {}
    for n_ in names:
        first.setdefault(n_, len(first))
    idx = sorted(range(len(keys)), key=lambda i: (first[names[i]], i))      # all_actions: by first-seen action name
    m = _model('dilated', seed=6).eval()
    for augment in (False, True):
        kw = dict(augment=augment, kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT,
                  thresholds=True)
        got = evaluate_sequences(m, p2, p3, groups, **kw)
        want = evaluate_sequences(m, [h2[o2[keys[i]]] for i in idx], [h3[order[keys[i]]] for i in idx],
                                  [names[i] for i in idx], **kw)
        assert got.groups == want.groups == ['Directions', 'Walking', 'Eating']
        for k in got.groups:
            a, b = got[k], want[k]
            assert (a.frames, a.mpjpe, a.p_mpjpe, a.pck, a.auc) == (b.frames, b.mpjpe, b.p_mpjpe, b.pck, b.auc)
            assert np.array_equal(a.per_joint, b.per_joint)


def test_generators_take_fetched_cuda_views():
    """DeviceSequences and UnchunkedGenerator concatenate / pad CUDA views (strided ones included) on the device and
    give what the same arrays give from the host"""
    from device.common.generators import UnchunkedGenerator
    ds_in, pos2d, g, meta = _standin('h36m')
    cams, p3, p2 = D.prepare(ds_in, pos2d).fetch(meta['fetch_subjects'], None, 5)
    host = [[x.cpu().numpy() for x in lst] for lst in (cams, p3, p2)]
    a, b = P.DeviceSequences(p2, p3, cams), P.DeviceSequences(host[2], host[1], host[0])
    assert all(torch.equal(getattr(a, k), getattr(b, k)) for k in ('seq_start', 'poses_2d', 'poses_3d', 'cameras'))
    kw = dict(pad=13, causal_shift=0, augment=True, kps_left=LEFT, kps_right=RIGHT, joints_left=LEFT, joints_right=RIGHT)
    for x, y in zip(UnchunkedGenerator(cams, p3, p2, **kw).next_epoch(), UnchunkedGenerator(*host, **kw).next_epoch()):
        assert all(torch.equal(u, v) for u, v in zip(x, y))
