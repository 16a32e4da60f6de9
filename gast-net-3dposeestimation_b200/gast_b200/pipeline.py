"""Device-resident versions of the steps either side of the lifting forward (SURVEY.md §8f N1-N3).

Each function takes and returns CUDA float32 tensors and launches one small kernel of
libgast_b200.so through the C ABI (include/gast_b200.h); the modules under `device/common/` and
`device/tools/` wrap them with the reference's own names and signatures.  No CPU path: a CPU tensor raises.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .engine import GastError, _call, _check_size, _cuda_f32, _ilist, _launch, _p

KPT_COCO_H36M, KPT_MPII_H36M, KPT_COCO_H36M_TOE, KPT_COCO_HUMANEVA = 0, 1, 2, 3


# ------------------------------------------------------------------------------------------------
# N1: training batches (common/generators.py:4-154)
# ------------------------------------------------------------------------------------------------
class DeviceSequences(object):
    """All videos of a dataset split concatenated along time in HBM: poses_2d (sum T,J2,F2), poses_3d
    (sum T,J3,3), cameras (n,ncam) and the prefix frame offsets -- what ChunkedGenerator indexes into
    (generators.py:64-66) once per batch on the host.  Lists of CUDA tensors (views included, as
    gast_b200.dataset's fetch returns them) are concatenated on the device."""

    def __init__(self, poses_2d, poses_3d=None, cameras=None, device='cuda'):
        lens = [int(p.shape[0]) for p in poses_2d]
        self.n_seq = len(lens)
        self.lengths = lens
        self.seq_start = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device=device)
        self.poses_2d = _joined(poses_2d, torch.cat, np.concatenate, device)
        self.poses_3d = None
        if poses_3d is not None:
            assert [int(p.shape[0]) for p in poses_3d] == lens
            self.poses_3d = _joined(poses_3d, torch.cat, np.concatenate, device)
        self.cameras = None
        if cameras is not None:
            self.cameras = _joined(cameras, torch.stack, np.stack, device)


def _joined(arrays, join_t, join_np, device):
    """the arrays joined along a new or the first axis as one float32 tensor on `device`: CUDA tensors on the device,
    anything else on the host and uploaded once"""
    if all(isinstance(a, torch.Tensor) and a.is_cuda for a in arrays):
        return join_t([a.to(device=device, dtype=torch.float32) for a in arrays], 0)
    return torch.as_tensor(join_np([np.asarray(a, dtype=np.float32) for a in arrays], 0)).to(device)


def chunk_gather(seqs, pairs, chunk_length, pad, causal_shift=0, kps_left=None, kps_right=None, joints_left=None,
                 joints_right=None):
    """One batch of ChunkedGenerator.next_epoch (generators.py:93-154).  pairs: (B,4) integer array of
    the reference's (seq_i, start_3d, end_3d, flip) tuples.  Returns (batch_cam, batch_3d, batch_2d) as
    CUDA float32 tensors (None where the split has no cameras / 3D poses)."""
    dev = seqs.poses_2d.device
    pr = torch.as_tensor(np.asarray(pairs, dtype=np.int64).astype(np.int32).reshape(-1, 4)).to(dev)
    B = int(pr.shape[0])
    J2, F2 = int(seqs.poses_2d.shape[1]), int(seqs.poses_2d.shape[2])
    b2 = torch.empty((B, chunk_length + 2 * pad, J2, F2), dtype=torch.float32, device=dev)
    b3, J3 = None, 0
    if seqs.poses_3d is not None:
        J3 = int(seqs.poses_3d.shape[1])
        b3 = torch.empty((B, chunk_length, J3, 3), dtype=torch.float32, device=dev)
    bc, ncam = None, 0
    if seqs.cameras is not None:
        ncam = int(seqs.cameras.shape[1])
        bc = torch.empty((B, ncam), dtype=torch.float32, device=dev)
    kl, n2 = _ilist(kps_left)
    kr, _ = _ilist(kps_right)
    jl, n3 = _ilist(joints_left)
    jr, _ = _ilist(joints_right)
    _launch(dev, 'gast_chunk_gather', _p(seqs.poses_2d), _p(seqs.poses_3d), _p(seqs.cameras), _p(seqs.seq_start),
            seqs.n_seq, _p(pr), B, int(chunk_length), int(pad), int(causal_shift), J2, F2, J3, ncam, n2, kl, kr, n3, jl,
            jr, _p(b2), _p(b3), _p(bc))
    return bc, b3, b2


def chunk_gather_indexed(seqs, pairs, batch, B, batch_stride, chunk_length, pad, causal_shift=0, kps_left=None,
                         kps_right=None, joints_left=None, joints_right=None):
    """chunk_gather of pairs[b*batch_stride : b*batch_stride + B], b the CUDA int64 batch counter `batch` (read on the
    device, so one CUDA graph serves every batch of an epoch).  pairs: the epoch's (n_pairs,4) CUDA int32 table.
    Same results, bit for bit; nothing is written when those rows are not all in the table."""
    dev = seqs.poses_2d.device
    if pairs.dtype != torch.int32 or pairs.dim() != 2 or pairs.shape[1] != 4 or not pairs.is_contiguous() \
            or batch.dtype != torch.int64 or pairs.device != dev or batch.device != dev:
        raise GastError('chunk_gather_indexed: pairs (n,4) contiguous int32 and an int64 batch counter on %s expected' % dev)
    J2, F2 = int(seqs.poses_2d.shape[1]), int(seqs.poses_2d.shape[2])
    b2 = torch.empty((B, chunk_length + 2 * pad, J2, F2), dtype=torch.float32, device=dev)
    b3, J3 = None, 0
    if seqs.poses_3d is not None:
        J3 = int(seqs.poses_3d.shape[1])
        b3 = torch.empty((B, chunk_length, J3, 3), dtype=torch.float32, device=dev)
    bc, ncam = None, 0
    if seqs.cameras is not None:
        ncam = int(seqs.cameras.shape[1])
        bc = torch.empty((B, ncam), dtype=torch.float32, device=dev)
    kl, n2 = _ilist(kps_left)
    kr, _ = _ilist(kps_right)
    jl, n3 = _ilist(joints_left)
    jr, _ = _ilist(joints_right)
    _launch(dev, 'gast_chunk_gather_indexed', _p(seqs.poses_2d), _p(seqs.poses_3d), _p(seqs.cameras),
            _p(seqs.seq_start), seqs.n_seq, _p(pairs), int(pairs.shape[0]), int(batch_stride), _p(batch), int(B),
            int(chunk_length), int(pad), int(causal_shift), J2, F2, J3, ncam, n2, kl, kr, n3, jl, jr, _p(b2), _p(b3),
            _p(bc))
    return bc, b3, b2


# ------------------------------------------------------------------------------------------------
# N3: keypoint formats, screen normalisation, camera -> world
# ------------------------------------------------------------------------------------------------
def keypoints_convert(kpts, mode):
    """tools/mpii_coco_h36m.py, and HumanEva's COCO -> 15 joints (main.py:80-95): (T,J_in,2) -> ((T,17|19|15,2), valid
    mask (T,) int32)."""
    k = _cuda_f32(kpts, 'keypoints_convert')
    if k.dim() != 3 or k.shape[-1] != 2:
        raise GastError('keypoints_convert: (T,J,2) expected')
    T, Jin = int(k.shape[0]), int(k.shape[1])
    Jo = {KPT_COCO_H36M_TOE: 19, KPT_COCO_HUMANEVA: 15}.get(mode, 17)
    out = torch.empty((T, Jo, 2), dtype=torch.float32, device=k.device)
    valid = torch.empty((T,), dtype=torch.int32, device=k.device)
    _launch(k.device, 'gast_keypoints_convert', _p(k), _p(out), _p(valid), T, Jin, int(mode))
    return out, valid


def normalize_screen(x, w, h, inverse=False):
    """common/camera.py:8-19 on (...,2) points."""
    x = _cuda_f32(x, 'normalize_screen')
    assert x.shape[-1] == 2
    out = torch.empty_like(x)
    _launch(x.device, 'gast_normalize_screen', _p(x), _p(out), x.numel() // 2, float(w), float(h), 1 if inverse else 0)
    return out


def camera_to_world(x, R, t=0):
    """common/camera.py:27-28 with one quaternion R (4,) and translation t (3,) or scalar for all points."""
    x = _cuda_f32(x, 'camera_to_world')
    assert x.shape[-1] == 3
    q = (C.c_float * 4)(*[float(v) for v in np.asarray(R, dtype=np.float32).reshape(4)])
    tv = np.broadcast_to(np.asarray(t, dtype=np.float32), (3,))
    tt = (C.c_float * 3)(*[float(v) for v in tv])
    out = torch.empty_like(x)
    _launch(x.device, 'gast_camera_to_world', _p(x), _p(out), x.numel() // 3, q, tt)
    return out


# ------------------------------------------------------------------------------------------------
# Dataset preparation (main.py:24-104, data/prepare_data_h36m.py:113-121): segmented launches.  Output segment s holds
# rows dst_start[s] .. dst_start[s+1]-1 taken from source rows src_start[s] ..; the tables are CUDA tensors (int64
# offsets, float32 / float64 parameters), so a launch reads nothing from the host.
# ------------------------------------------------------------------------------------------------
def _table(t, dtype, shape, dev, what):
    if not isinstance(t, torch.Tensor) or t.dtype != dtype or tuple(t.shape) != tuple(shape) or t.device != dev \
            or not t.is_contiguous():
        raise GastError('%s: a contiguous %s table %s on %s expected, got %s' % (
            what, dtype, tuple(shape), dev, (t.dtype, tuple(t.shape), t.device) if isinstance(t, torch.Tensor) else type(t)))
    return t


def world_to_camera_segments(x, src_start, dst_start, qt, n_out, root_relative=False):
    """world_to_camera (camera.py:22-24) of frames x (n_src,J,3) -> (n_out,J,3): segment s from its own source frames
    with qt[s] = {orientation[4], translation[3]}; root_relative also does main.py:33 (pos[:, 1:] -= pos[:, :1])."""
    x = _cuda_f32(x, 'world_to_camera')
    if x.dim() != 3 or x.shape[-1] != 3:
        raise GastError('world_to_camera: frames (n,J,3) expected, got %s' % (tuple(x.shape),))
    S, dev = int(qt.shape[0]) if isinstance(qt, torch.Tensor) else 0, x.device
    _table(qt, torch.float32, (S, 7), dev, 'world_to_camera')
    _table(src_start, torch.int64, (S,), dev, 'world_to_camera')
    _table(dst_start, torch.int64, (S + 1,), dev, 'world_to_camera')
    out = torch.empty((int(n_out), int(x.shape[1]), 3), dtype=torch.float32, device=dev)
    _launch(dev, 'gast_world_to_camera', _p(x), int(x.shape[0]), int(x.shape[1]), _p(src_start), _p(dst_start), _p(qt),
            S, int(n_out), 1 if root_relative else 0, _p(out))
    return out


def world_to_camera(x, R, t):
    """camera.py:22-24 with one rotation R (4,) and translation t (3,) for every point of x (...,3); R and t may be
    host arrays or tensors on any device"""
    x = _cuda_f32(x, 'world_to_camera')
    assert x.shape[-1] == 3
    dev = x.device
    qt = torch.cat([torch.as_tensor(R, dtype=torch.float32).reshape(4).to(dev),
                    torch.as_tensor(t, dtype=torch.float32).reshape(3).to(dev)]).reshape(1, 7)
    n = x.numel() // 3
    offs = torch.tensor([0, 0, n], dtype=torch.int64, device=dev)           # src_start = {0}, dst_start = {0, n}
    return world_to_camera_segments(x.reshape(n, 1, 3), offs[:1], offs[1:], qt, n).reshape(x.shape)


def project_to_2d_segments(x, seg_start, intrinsics, grad_out=None):
    """project_to_2d (camera.py:31-62) of the points x (...,3) -> (...,2); the points seg_start[s] .. seg_start[s+1]-1
    (in points) use intrinsics[s] (9,).  With grad_out (...,2) returns dL/dx (...,3) instead."""
    x = _cuda_f32(x, 'project_to_2d')
    if x.shape[-1] != 3:
        raise GastError('project_to_2d: points (...,3) expected, got %s' % (tuple(x.shape),))
    dev, n = x.device, x.numel() // 3
    S = int(intrinsics.shape[0]) if isinstance(intrinsics, torch.Tensor) else 0
    _table(intrinsics, torch.float32, (S, 9), dev, 'project_to_2d')
    _table(seg_start, torch.int64, (S + 1,), dev, 'project_to_2d')
    if grad_out is None:
        out = torch.empty(tuple(x.shape[:-1]) + (2,), dtype=torch.float32, device=dev)
        _launch(dev, 'gast_project_to_2d', _p(x), n, _p(seg_start), _p(intrinsics), S, _p(out))
    else:
        g = _cuda_f32(grad_out, 'project_to_2d backward')
        if tuple(g.shape) != tuple(x.shape[:-1]) + (2,):
            raise GastError('project_to_2d backward: grad (...,2) of the points expected, got %s' % (tuple(g.shape),))
        out = torch.empty_like(x)
        _launch(dev, 'gast_project_to_2d_backward', _p(x), n, _p(seg_start), _p(intrinsics), S, _p(g), _p(out))
    return out


def normalize_screen_segments(x, src_start, dst_start, wh, n_out, from_image=False):
    """normalize_screen_coordinates (camera.py:8-12) of frames x (n_src,P,F>=2) -> (n_out,P,F): channels 0 and 1 with
    segment s's wh[s] = {w, h/w} (float64), the others copied.  from_image first takes the points through
    image_coordinates and float32 (the ground-truth keypoints' round trip)."""
    x = _cuda_f32(x, 'normalize_screen_segments')
    if x.dim() != 3 or x.shape[-1] < 2:
        raise GastError('normalize_screen_segments: frames (n,P,F>=2) expected, got %s' % (tuple(x.shape),))
    S = int(wh.shape[0]) if isinstance(wh, torch.Tensor) else 0
    dev = x.device
    _table(wh, torch.float64, (S, 2), dev, 'normalize_screen_segments')
    _table(src_start, torch.int64, (S,), dev, 'normalize_screen_segments')
    _table(dst_start, torch.int64, (S + 1,), dev, 'normalize_screen_segments')
    P, F = int(x.shape[1]), int(x.shape[2])
    out = torch.empty((int(n_out), P, F), dtype=torch.float32, device=dev)
    _launch(dev, 'gast_normalize_screen_segments', _p(x), int(x.shape[0]), P, F, _p(src_start), _p(dst_start), _p(wh),
            S, int(n_out), 1 if from_image else 0, _p(out))
    return out


# ------------------------------------------------------------------------------------------------
# The video demo's keypoint repair and placement of the lifted persons (tools/preprocess.py)
# ------------------------------------------------------------------------------------------------
def _prep_ws(dev, nbytes):
    """the call's own scratch (placement minima, metric partials) from the caching allocator, freed to the current
    stream when the call returns: a scratch kept across calls would be shared by calls in flight on two streams and
    freed under a call still queued on another stream or captured in a CUDA graph"""
    return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


def h36m_coco_format(kpts, scores):
    """preprocess.py:47-75 over every person slot: kpts (P,T,17,2), scores (P,T,17) -> (H36M keypoints (P,T,17,2),
    H36M scores (P,T,17), valid mask (P,T) int32, keep (P,) int32).  The caller drops the slots whose keep is 0."""
    k = _cuda_f32(kpts, 'h36m_coco_format')
    s = _cuda_f32(scores, 'h36m_coco_format')
    if k.dim() != 4 or tuple(k.shape[2:]) != (17, 2) or tuple(s.shape) != tuple(k.shape[:3]):
        raise GastError('h36m_coco_format: kpts (P,T,17,2) and scores (P,T,17) expected, got %s and %s'
                        % (tuple(k.shape), tuple(s.shape)))
    P, T = int(k.shape[0]), int(k.shape[1])
    dev = k.device
    out = torch.empty_like(k)
    sout = torch.empty_like(s)
    valid = torch.empty((P, T), dtype=torch.int32, device=dev)
    keep = torch.empty((P,), dtype=torch.int32, device=dev)
    _launch(dev, 'gast_h36m_coco_format', _p(k), _p(s), P, T, _p(out), _p(sout), _p(valid), _p(keep))
    return out, sout, valid, keep


def revise_kpts(kpts, scores, valid):
    """preprocess.py:78-112: kpts (P,T,J,2), scores (P,T,J), valid (P,T) int32 mask -> repaired kpts (P,T,J,2)."""
    k = _cuda_f32(kpts, 'revise_kpts')
    s = _cuda_f32(scores, 'revise_kpts')
    if k.dim() != 4 or k.shape[-1] != 2 or tuple(s.shape) != tuple(k.shape[:3]) or tuple(valid.shape) != tuple(k.shape[:2]):
        raise GastError('revise_kpts: kpts (P,T,J,2), scores (P,T,J) and valid (P,T) expected')
    v = valid.to(torch.int32).contiguous()
    P, T, J = (int(d) for d in k.shape[:3])
    out = torch.empty_like(k)
    _launch(k.device, 'gast_revise_kpts', _p(k), _p(s), _p(v), P, T, J, _p(out))
    return out


def revise_skes(pred, frames, offsets, kpts):
    """preprocess.py:123-155: pred (N,J,3) every person's prediction packed (person p at rows offsets[p] ..
    offsets[p+1]-1; offsets a host sequence of P+1 ints), frames (N,) CUDA int64 the frame of each row, kpts (P,T,J,D)
    -> (P,T,J,3).  Two persons without a common frame get NaN x and y (the caller checks host frame lists)."""
    pr = _cuda_f32(pred, 'revise_skes')
    k = _cuda_f32(kpts, 'revise_skes')
    fr = frames.contiguous()
    off = np.ascontiguousarray(offsets, dtype=np.int64)
    if k.dim() != 4 or pr.dim() != 3 or pr.shape[-1] != 3 or pr.shape[1] != k.shape[2] or fr.dtype != torch.int64 \
            or not fr.is_cuda or off.shape != (k.shape[0] + 1,) or int(off[-1]) != pr.shape[0] or fr.numel() != pr.shape[0]:
        raise GastError('revise_skes: pred (N,J,3), frames (N,) CUDA int64, offsets (P+1,) and kpts (P,T,J,D) expected')
    P, T, J, D = (int(d) for d in k.shape)
    dev = k.device
    out = torch.empty((P, T, J, 3), dtype=torch.float32, device=dev)
    ws = _prep_ws(dev, L.load().gast_revise_skes_workspace_bytes(P, T))
    _launch(dev, 'gast_revise_skes', _p(pr), _p(fr), off.ctypes.data_as(C.POINTER(C.c_int64)), P, T, J, D, _p(k),
            _p(out), _p(ws), ws.numel())
    return out


def revise_skes_real_time(pred, kpts, width):
    """preprocess.py:158-172: pred (M,17,3), kpts (M,17,D) of one tick, image width -> placed poses (M,17,3)."""
    pr = _cuda_f32(pred, 'revise_skes_real_time')
    k = _cuda_f32(kpts, 'revise_skes_real_time')
    if pr.dim() != 3 or pr.shape[-1] != 3 or k.dim() != 3 or k.shape[0] != pr.shape[0] or k.shape[1] != pr.shape[1]:
        raise GastError('revise_skes_real_time: pred (M,17,3) and kpts (M,17,D) expected, got %s and %s'
                        % (tuple(pr.shape), tuple(k.shape)))
    M, J, D = int(pr.shape[0]), int(pr.shape[1]), int(k.shape[2])
    dev = pr.device
    out = torch.empty_like(pr)
    ws = _prep_ws(dev, L.load().gast_revise_skes_real_time_workspace_bytes(M))
    _launch(dev, 'gast_revise_skes_real_time', _p(pr), _p(k), M, J, D, float(width), _p(out), _p(ws), ws.numel())
    return out


# ------------------------------------------------------------------------------------------------
# N2: losses and the optimiser step
# ------------------------------------------------------------------------------------------------
def _mpjpe_ws(dev):
    """the call's own block partials (see _prep_ws)"""
    return torch.empty(int(L.load().gast_mpjpe_workspace_bytes()), dtype=torch.uint8, device=dev)


class _MpjpeFn(torch.autograd.Function):
    """loss and d loss / d predicted from one pass over the data (common/loss.py:5-11)."""

    @staticmethod
    def forward(ctx, predicted, target):
        p = _cuda_f32(predicted, 'mpjpe')
        t = _cuda_f32(target, 'mpjpe')
        D = int(p.shape[-1])
        loss = torch.empty((), dtype=torch.float32, device=p.device)
        need = predicted.requires_grad
        dp = torch.empty_like(p) if need else None
        _launch(p.device, 'gast_mpjpe', _p(p), _p(t), p.numel() // D, D, _p(loss), _p(dp), 1.0, _p(_mpjpe_ws(p.device)))
        if need:
            ctx.save_for_backward(dp)
        return loss

    @staticmethod
    def backward(ctx, g):
        (dp,) = ctx.saved_tensors
        return dp * g, None


def mpjpe(predicted, target):
    assert predicted.shape == target.shape
    return _MpjpeFn.apply(predicted, target)


def p_mpjpe_per_frame(predicted, target):
    """(N,J,3) x2 -> (N,) mean joint error after Procrustes alignment (common/loss.py:14-53)."""
    p = _cuda_f32(predicted, 'p_mpjpe')
    t = _cuda_f32(target, 'p_mpjpe')
    assert p.shape == t.shape and p.dim() == 3 and p.shape[-1] == 3
    N, J = int(p.shape[0]), int(p.shape[1])
    out = torch.empty((N,), dtype=torch.float32, device=p.device)
    _launch(p.device, 'gast_p_mpjpe', _p(p), _p(t), N, J, _p(out))
    return out


def pose_metrics(predicted, target, seg_start, thresholds=(), zero_root=False, procrustes=True, distances=False):
    """Score rows per segment (gast_pose_metrics; main.py:299-353, common/loss.py:56-90).  predicted, target (N,J,3)
    CUDA float32; seg_start the S+1 host frame offsets of the segments, 0 .. N; thresholds host floats (compared in
    float32, as torch compares a float32 tensor with a Python float).  Returns the (S, 3+J+n_thr) float64 CUDA tensor
    [frames, sum_f mpjpe_f, sum_f p_mpjpe_f (0 without procrustes), sum_f dist_fj (J), count(dist < thr_k) (n_thr)],
    and with distances=True also the (N,J) float32 joint distances.  zero_root reads target joint 0 as 0 without
    writing the target.  Every argument is checked before the first launch."""
    p = _cuda_f32(predicted, 'pose_metrics')
    t = _cuda_f32(target, 'pose_metrics')
    if p.shape != t.shape or p.dim() != 3 or p.shape[-1] != 3 or p.device != t.device:
        raise GastError('pose_metrics: predicted and target (N,J,3) on one device expected, got %s and %s'
                        % (tuple(p.shape), tuple(t.shape)))
    seg = np.ascontiguousarray(np.asarray(seg_start, dtype=np.int64).reshape(-1))
    thr = np.ascontiguousarray(np.asarray(thresholds, dtype=np.float32).reshape(-1))
    N, J, S = int(p.shape[0]), int(p.shape[1]), int(seg.size) - 1
    dev = p.device
    wb = _check_size(L.load().gast_pose_metrics_workspace_bytes(S, J, int(thr.size), N), 'pose_metrics')
    rows = torch.empty((S, 3 + J + int(thr.size)), dtype=torch.float64, device=dev)
    dist = torch.empty((N, J), dtype=torch.float32, device=dev) if distances else None
    ws = _prep_ws(dev, wb)
    _launch(dev, 'gast_pose_metrics', _p(p), _p(t), N, J, seg.ctypes.data_as(C.POINTER(C.c_int64)), S,
            thr.ctypes.data_as(C.POINTER(C.c_float)), int(thr.size), 1 if zero_root else 0, 1 if procrustes else 0,
            _p(rows), _p(dist), _p(ws), ws.numel())
    return (rows, dist) if distances else rows


def adam_step_table(lr, betas, first_step, n_steps):
    """(n_steps,2) float32 numpy: {lr / bc1, sqrt(bc2)} of steps first_step .. first_step + n_steps - 1, rounded as
    gast_adam_step rounds them (gast_adam_step_table), for FusedAdam.step_indexed."""
    out = np.empty((int(n_steps), 2), dtype=np.float32)
    _call('gast_adam_step_table', float(lr), float(betas[0]), float(betas[1]), int(first_step), int(n_steps),
          out.ctypes.data_as(C.c_void_p))
    return out


def epoch_loss_accumulate(loss, weight, loss_sum, losses, batch):
    """The last launch of an epoch step: losses[b] = loss, loss_sum += weight * loss in fp64, b += 1 (b the CUDA int64
    batch counter `batch`).  loss 0-d float32, loss_sum 0-d float64, losses (n_steps,) float32, all on one device."""
    dev = loss.device
    if loss.dtype != torch.float32 or loss_sum.dtype != torch.float64 or losses.dtype != torch.float32 \
            or batch.dtype != torch.int64 or {loss_sum.device, losses.device, batch.device} != {dev} or not loss.is_cuda:
        raise GastError('epoch_loss_accumulate: float32 loss, float64 sum, float32 losses and an int64 batch counter '
                        'on one CUDA device expected')
    _launch(dev, 'gast_epoch_loss_accumulate', _p(loss), int(weight), _p(loss_sum), _p(losses), losses.numel(),
            _p(batch))


class FusedAdam(object):
    """optim.Adam(params, lr, amsgrad=True) (trainval.py:78) as ONE kernel launch per step over every
    parameter (the stock optimiser issues ~10 elementwise launches per tensor, ~2000 per step here).
    The moments live in three flat buffers; parameters and gradients stay where they are and are
    reached through a device table of (param ptr, grad ptr, state offset, count) chunks.  `param_groups`
    mirrors torch's so that trainval.py:162-164's `param_group['lr'] *= lr_decay` works unchanged."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, amsgrad=False):
        self.params = [p for p in params if p.requires_grad]
        if not self.params or not all(p.is_cuda and p.dtype == torch.float32 for p in self.params):
            raise GastError('FusedAdam: CUDA float32 parameters required')
        self.param_groups = [{'params': self.params, 'lr': lr, 'betas': betas, 'eps': eps, 'weight_decay': weight_decay,
                              'amsgrad': amsgrad}]
        dev = self.params[0].device
        n = sum(p.numel() for p in self.params)
        self.exp_avg = torch.zeros(n, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev)
        self.max_exp_avg_sq = torch.zeros(n, dtype=torch.float32, device=dev) if amsgrad else None
        self.step_count = 0
        self._sig = None
        self._table = None

    def zero_grad(self, set_to_none=False):
        for p in self.params:
            if p.grad is not None:
                p.grad.zero_()

    def _build_table(self):
        sig = tuple((p.data_ptr(), p.grad.data_ptr()) for p in self.params)
        if sig == self._sig:
            return
        chunk = int(L.load().gast_adam_chunk())
        rows, off = [], 0
        for p in self.params:
            if not p.is_contiguous() or not p.grad.is_contiguous():
                raise GastError('FusedAdam: contiguous parameters and gradients required')
            n = p.numel()
            for c0 in range(0, n, chunk):
                rows.append((p.data_ptr() + 4 * c0, p.grad.data_ptr() + 4 * c0, off + c0, min(chunk, n - c0)))
            off += n
        self._table = torch.tensor(rows, dtype=torch.int64, device=self.params[0].device)
        self._sig = sig

    def step(self):
        if any(p.grad is None for p in self.params):
            raise GastError('FusedAdam.step: every parameter needs a gradient')
        self._build_table()
        g = self.param_groups[0]
        self.step_count += 1
        dev = self.params[0].device
        _launch(dev, 'gast_adam_step', _p(self._table), int(self._table.shape[0]), _p(self.exp_avg),
                _p(self.exp_avg_sq), _p(self.max_exp_avg_sq), float(g['lr']), float(g['betas'][0]),
                float(g['betas'][1]), float(g['eps']), float(g['weight_decay']), self.step_count)
        # the kernel writes the parameters through raw pointers: bump their version counters so that everything
        # keyed on (data_ptr, _version) -- the engine's folded eval-mode constants -- sees the update
        torch.autograd.graph.increment_version(self.params)

    def step_indexed(self, coef, batch):
        """step() at step step_count + 1 + b without a host argument that changes per step: b the CUDA int64 batch
        counter `batch`, coef the (n_steps,2) CUDA float32 adam_step_table of the steps from step_count + 1 at the
        current lr.  Bit for bit step()'s update; no update when b >= n_steps.  step_count is the caller's to
        advance (EpochTrainer adds an epoch's steps at its end)."""
        if any(p.grad is None for p in self.params):
            raise GastError('FusedAdam.step_indexed: every parameter needs a gradient')
        dev = self.params[0].device
        if coef.dtype != torch.float32 or coef.dim() != 2 or coef.shape[1] != 2 or not coef.is_contiguous() \
                or batch.dtype != torch.int64 or coef.device != dev or batch.device != dev:
            raise GastError('FusedAdam.step_indexed: coef (n,2) contiguous float32 and an int64 batch counter on %s '
                            'expected' % dev)
        self._build_table()
        g = self.param_groups[0]
        _launch(dev, 'gast_adam_step_indexed', _p(self._table), int(self._table.shape[0]), _p(self.exp_avg),
                _p(self.exp_avg_sq), _p(self.max_exp_avg_sq), float(g['betas'][0]), float(g['betas'][1]),
                float(g['eps']), float(g['weight_decay']), _p(coef), int(coef.shape[0]), _p(batch))
        torch.autograd.graph.increment_version(self.params)

    def state_dict(self):
        return {'step': self.step_count, 'exp_avg': self.exp_avg, 'exp_avg_sq': self.exp_avg_sq,
                'max_exp_avg_sq': self.max_exp_avg_sq, 'param_groups': [{k: v for k, v in g.items() if k != 'params'}
                                                                       for g in self.param_groups]}

    def load_state_dict(self, sd):
        self.step_count = int(sd['step'])
        self.exp_avg.copy_(sd['exp_avg'])
        self.exp_avg_sq.copy_(sd['exp_avg_sq'])
        if self.max_exp_avg_sq is not None and sd.get('max_exp_avg_sq') is not None:
            self.max_exp_avg_sq.copy_(sd['max_exp_avg_sq'])
        for g, s in zip(self.param_groups, sd['param_groups']):
            g.update(s)
