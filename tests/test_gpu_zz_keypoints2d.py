"""The 2D pose net's crop and heatmap decode on the device (gast_b200.keypoints2d, csrc/keypoints2d.cuh) against the
reference's outputs (tests/golden/keypoints2d.npz) and the numpy restatement (tests/keypoints2dref.py), bit for bit.
The matrices come from the goldens, so the tests need no cv2."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import keypoints2dref as R                                          # noqa: E402
from conftest import load_golden                                    # noqa: E402
from gast_b200 import keypoints2d as K                              # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def gold():
    g = load_golden('keypoints2d')
    m = g['meta']
    g['frames'] = R.synth_frames(m['F'], m['H'], m['W'])
    return g


def bits_equal(a, b):
    a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, np.float32)
    b = b.cpu().numpy() if isinstance(b, torch.Tensor) else np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


@pytest.mark.parametrize('net_order', [True, False])
@pytest.mark.parametrize('rgb', [False, True])
def test_crops_equal_the_reference_warps(gold, net_order, rgb):
    """every box of three frames in one call, both plane orders, BGR and RGB frames"""
    m = gold['meta']
    frames = torch.from_numpy(gold['frames']).cuda()
    if rgb:
        frames = frames.flip(-1).contiguous()
    out = K.crop_persons(frames, gold['box_frame'], gold['fwd_small'], m['small'], rgb_input=rgb, net_order=net_order)
    assert out.shape == (len(gold['boxes']), 3, m['small'][1], m['small'][0]) and out.dtype == torch.float32
    for k in range(len(gold['boxes'])):
        assert bits_equal(out[k], R.normalize(gold['warps_small'][k], net_order=net_order)), k
    # w48_384x288's crop size: the stored cv2 warps, and every box against the restatement of cv2's warp
    full = K.crop_persons(frames, gold['box_frame'], gold['fwd_full'], m['full'], rgb_input=rgb, net_order=net_order)
    for k in range(len(gold['boxes'])):
        f = gold['frames'][gold['box_frame'][k]]
        assert bits_equal(full[k], R.crop(f, gold['fwd_full'][k], m['full'], net_order=net_order)), k
        if k < m['full_n']:
            assert bits_equal(full[k], R.normalize(gold['warps_full'][k], net_order=net_order)), k


@pytest.mark.parametrize('size', [(72, 96), (48, 64)])
@pytest.mark.parametrize('post', [True, False])
def test_decode_equals_the_reference(gold, size, post):
    hw, hh = size
    hm = np.concatenate([R.edge_case_heatmaps(hh, hw), R.synth_heatmaps(4, 17, hh, hw, seed=3)])
    key = 'dec_%dx%d_%s' % (hw, hh, 'post' if post else 'plain')
    p, mv = K.decode_heatmaps(torch.from_numpy(hm).cuda(), gold['inv_%dx%d' % size][:hm.shape[0]], post)
    assert p.is_cuda and bits_equal(p, gold[key + '_preds']) and bits_equal(mv, gold[key + '_maxvals'])


def test_preprocess_drop_in(gold):
    """PreProcess: numpy and CUDA frames give the reference's inputs (bit for bit with cv2's matrices; without cv2
    the closed-form matrices' own warp), centers and scales"""
    from device.lib.pose.hrnet.lib.utils.utilitys import PreProcess
    m = gold['meta']
    cfg = SimpleNamespace(MODEL=SimpleNamespace(IMAGE_SIZE=list(m['pre_size'])))
    for i, (f, b0, nb, num_pos) in enumerate(m['pre_calls']):
        boxes = [list(r) for r in gold['boxes'][b0:b0 + nb]]
        frame = gold['frames'][f]
        for img in (frame, torch.from_numpy(frame).cuda()):
            inputs, back, c, s = PreProcess(img, boxes, cfg, num_pos)
            assert back is img and inputs.is_cuda
            assert bits_equal(np.stack(c), gold['pre%d_centers' % i]) and bits_equal(np.stack(s), gold['pre%d_scales' % i])
            if K._cv2 is not None:
                want = gold['pre%d_inputs' % i]
            else:
                want = np.stack([R.crop(frame, K.affine_pair(ci, si, m['pre_size'])[0], m['pre_size'], net_order=False)
                                 for ci, si in zip(c, s)])
            assert bits_equal(inputs, want), i


def test_get_final_preds_drop_in(gold):
    from device.lib.pose.hrnet.lib.utils.inference import get_final_preds
    hw, hh = 72, 96
    hm = np.concatenate([R.edge_case_heatmaps(hh, hw), R.synth_heatmaps(4, 17, hh, hw, seed=3)])
    n = hm.shape[0]
    for post in (True, False):
        cfg = SimpleNamespace(TEST=SimpleNamespace(POST_PROCESS=post))
        key = 'dec_%dx%d_%s' % (hw, hh, 'post' if post else 'plain')
        if K._cv2 is not None:
            want = gold[key + '_preds']
        else:
            inv = [K.inverse_matrix(gold['centers'][i], gold['scales'][i], (hw, hh)) for i in range(n)]
            want = R.decode(hm, inv, post)[0]
        p, mv = get_final_preds(cfg, hm, gold['centers'][:n], gold['scales'][:n])
        assert isinstance(p, np.ndarray) and p.dtype == np.float32 and bits_equal(p, want)
        assert bits_equal(mv, gold[key + '_maxvals'])
        pc, mvc = get_final_preds(cfg, torch.from_numpy(hm).cuda(), gold['centers'][:n], gold['scales'][:n])
        assert pc.is_cuda and bits_equal(pc, p) and bits_equal(mvc, mv)


class _StandInNet(torch.nn.Module):
    """a seeded stand-in for HRNet, (n, 3, 384, 288) -> (n, 17, 96, 72): a 4 x 4 average pool and a per-joint mix of
    the planes through a sine.  Every output depends on its own crop only, whatever the batch, so split chunks can be
    compared byte for byte.  Records its inputs and heatmaps."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        self.register_buffer('w', torch.rand((17, 3), generator=g) * 4 - 2)
        self.register_buffer('b', torch.rand(17, generator=g) * 6)
        self.seen = []

    def forward(self, x):
        p = torch.nn.functional.avg_pool2d(x, 4)
        y = torch.stack([torch.sin(p[:, 0] * self.w[j, 0] + p[:, 1] * self.w[j, 1] + p[:, 2] * self.w[j, 2] + self.b[j])
                         for j in range(17)], 1)
        self.seen.append((x.clone(), y.clone()))
        return y


def _clip():
    T, H, W = 6, 540, 960
    frames = R.synth_frames(T, H, W, seed=2)
    tr = lambda *rows: np.array([list(r) + [i + 1] for i, r in enumerate(rows)], np.float64)  # noqa: E731
    boxes = [tr([100.123, 50.2, 300.7, 500.1], [600.0, 80.5, 790.25, 530.0]),
             None,
             tr([400.5, 100.0, 560.0, 520.3]),
             tr([-30.0, 20.0, 150.0, 400.0], [700.0, 300.0, 1000.0, 600.0], [300.0, 10.0, 480.0, 470.0]),
             np.zeros((0, 5)),
             tr([200.0, 60.0, 380.0, 510.0], [650.0, 70.0, 820.0, 525.0])]
    return frames, boxes


def _expected(frames, boxes, net, num_person):
    """the restatement on the net's own crops and heatmaps, laid out as gen_video_kpts lays them out"""
    H, W = frames.shape[1:3]
    crops, heat = net.seen[-1]
    crops, heat = crops.cpu().numpy(), heat.cpu().numpy()
    kept = [(t, K.select_tracks(b, num_person)) for t, b in enumerate(boxes) if K.select_tracks(b, num_person) is not None]
    kp = np.zeros((num_person, len(kept), 17, 2), np.float32)
    sc = np.zeros((num_person, len(kept), 17), np.float32)
    r = 0
    for to, (t, rows) in enumerate(kept):
        for p, box in enumerate(rows[:num_person]):
            c, s = K.center_scale(box, H, W)
            assert bits_equal(crops[r], R.crop(frames[t], K.affine_pair(c, s)[0], K.IMAGE_SIZE)), (t, p)
            pr, mv = R.decode(heat[r:r + 1], [K.inverse_matrix(c, s, (72, 96))], True)
            kp[p, to], sc[p, to] = pr[0], mv[0, :, 0]
            r += 1
    assert r == crops.shape[0]
    return kp, sc


@pytest.mark.parametrize('num_person', [2, 1])
def test_video_keypoints_equal_the_restatement(num_person):
    """dropped frames, a lone track kept with num_person = 2, the last num_person tracks reversed; and the chain into
    h36m_coco_format"""
    from device.tools.preprocess import h36m_coco_format
    frames, boxes = _clip()
    net = _StandInNet().cuda()
    kp, sc = K.video_keypoints(torch.from_numpy(frames).cuda(), boxes, net, num_person)
    assert kp.shape == (num_person, 4, 17, 2) and sc.shape == (num_person, 4, 17)
    ekp, esc = _expected(frames, boxes, net, num_person)
    assert bits_equal(kp, ekp) and bits_equal(sc, esc)
    if num_person == 2:
        assert not kp[1, 1].any() and kp[1, 0].any()                # the lone track of frame 2 leaves slot 1 zero
    hk, hs, valid = h36m_coco_format(kp, sc)
    nk, ns, nvalid = h36m_coco_format(ekp, esc)
    assert bits_equal(hk, nk) and bits_equal(hs, ns)
    # numpy frames and RGB frames give the same bytes
    kp2, sc2 = K.video_keypoints(frames, boxes, net, num_person)
    kp3, sc3 = K.video_keypoints(np.ascontiguousarray(frames[..., ::-1]), boxes, net, num_person, rgb_input=True)
    assert torch.equal(kp2, kp) and torch.equal(sc2, sc) and torch.equal(kp3, kp) and torch.equal(sc3, sc)


def test_split_and_repeated_calls_give_the_same_bytes(gold):
    m = gold['meta']
    frames = torch.from_numpy(gold['frames']).cuda()
    whole = K.crop_persons(frames, gold['box_frame'], gold['fwd_small'], m['small'])
    a = K.crop_persons(frames, gold['box_frame'][:5], gold['fwd_small'][:5], m['small'])
    b = K.crop_persons(frames, gold['box_frame'][5:], gold['fwd_small'][5:], m['small'])
    assert torch.equal(torch.cat([a, b]), whole)
    later = np.nonzero(gold['box_frame'] >= 1)[0]                  # the same records cut from fewer frames
    c = K.crop_persons(frames[1:], gold['box_frame'][later] - 1, gold['fwd_small'][later], m['small'])
    assert torch.equal(c, whole[torch.from_numpy(later).cuda()])
    assert torch.equal(K.crop_persons(frames, gold['box_frame'], gold['fwd_small'], m['small']), whole)
    hm = torch.from_numpy(R.synth_heatmaps(16, 17, 96, 72, seed=9)).cuda()
    p, mv = K.decode_heatmaps(hm, gold['inv_72x96'])
    p1, mv1 = K.decode_heatmaps(hm[:7], gold['inv_72x96'][:7])
    p2, mv2 = K.decode_heatmaps(hm[7:], gold['inv_72x96'][7:])
    assert torch.equal(torch.cat([p1, p2]), p) and torch.equal(torch.cat([mv1, mv2]), mv)
    q, qv = K.decode_heatmaps(hm, gold['inv_72x96'])
    assert torch.equal(q, p) and torch.equal(qv, mv)
    frames_np, boxes = _clip()
    net = _StandInNet().cuda()
    whole_kp, whole_sc = K.video_keypoints(frames_np, boxes, net, 2)
    k1, s1 = K.video_keypoints(frames_np[:3], boxes[:3], net, 2)
    k2, s2 = K.video_keypoints(frames_np[3:], boxes[3:], net, 2)
    assert torch.equal(torch.cat([k1, k2], 1), whole_kp) and torch.equal(torch.cat([s1, s2], 1), whole_sc)


def test_no_host_synchronisation(gold):
    m = gold['meta']
    frames = torch.from_numpy(gold['frames']).cuda()
    hm = torch.from_numpy(R.synth_heatmaps(16, 17, 96, 72, seed=9)).cuda()
    frames_np, boxes = _clip()
    dframes = torch.from_numpy(frames_np).cuda()
    net = _StandInNet().cuda()
    K.video_keypoints(dframes, boxes, net, 2)                       # warm up the net's kernels
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        c = K.crop_persons(frames, gold['box_frame'], gold['fwd_small'], m['small'])
        p, mv = K.decode_heatmaps(hm, gold['inv_72x96'])
        kp, sc = K.video_keypoints(dframes, boxes, net, 2)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert c.shape[0] == 16 and p.shape == (16, 17, 2) and kp.shape == (2, 4, 17, 2)
