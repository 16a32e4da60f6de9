"""Device-resident versions of the steps either side of the lifting forward (SURVEY.md §8f N1-N3).

Each function takes and returns CUDA float32 tensors and launches one small kernel of
libgast_b200.so through the C ABI (include/gast_b200.h); the modules under `device/common/` and
`device/tools/` wrap them with the reference's own names and signatures.  No CPU path: a CPU tensor raises.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib as L
from .engine import GastError, _check, _stream

KPT_COCO_H36M, KPT_MPII_H36M, KPT_COCO_H36M_TOE = 0, 1, 2


def _ilist(v):
    v = [] if v is None else list(v)
    return (C.c_int32 * max(len(v), 1))(*[int(i) for i in v]), len(v)


def _cuda_f32(x, what):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise GastError('%s: a CUDA tensor is required (there is no CPU path)' % what)
    if x.dtype != torch.float32:
        raise GastError('%s: float32 expected, got %s' % (what, x.dtype))
    return x.contiguous()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


# ------------------------------------------------------------------------------------------------
# N1: training batches (common/generators.py:4-154)
# ------------------------------------------------------------------------------------------------
class DeviceSequences(object):
    """All videos of a dataset split concatenated along time in HBM: poses_2d (sum T,J2,F2), poses_3d
    (sum T,J3,3), cameras (n,ncam) and the prefix frame offsets -- what ChunkedGenerator indexes into
    (generators.py:64-66) once per batch on the host."""

    def __init__(self, poses_2d, poses_3d=None, cameras=None, device='cuda'):
        lens = [int(p.shape[0]) for p in poses_2d]
        self.n_seq = len(lens)
        self.lengths = lens
        self.seq_start = torch.tensor(np.concatenate([[0], np.cumsum(lens)]), dtype=torch.int64, device=device)
        self.poses_2d = torch.as_tensor(np.concatenate([np.asarray(p, dtype=np.float32) for p in poses_2d], 0)).to(device)
        self.poses_3d = None
        if poses_3d is not None:
            assert [int(p.shape[0]) for p in poses_3d] == lens
            self.poses_3d = torch.as_tensor(np.concatenate([np.asarray(p, dtype=np.float32) for p in poses_3d], 0)).to(device)
        self.cameras = None
        if cameras is not None:
            self.cameras = torch.as_tensor(np.stack([np.asarray(c, dtype=np.float32) for c in cameras], 0)).to(device)


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
    with torch.cuda.device(dev):
        _check(L.load().gast_chunk_gather(_p(seqs.poses_2d), _p(seqs.poses_3d), _p(seqs.cameras), _p(seqs.seq_start),
                                          seqs.n_seq, _p(pr), B, int(chunk_length), int(pad), int(causal_shift), J2, F2,
                                          J3, ncam, n2, kl, kr, n3, jl, jr, _p(b2), _p(b3), _p(bc),
                                          C.c_void_p(_stream(dev))), 'gast_chunk_gather')
    return bc, b3, b2


# ------------------------------------------------------------------------------------------------
# N3: keypoint formats, screen normalisation, camera -> world
# ------------------------------------------------------------------------------------------------
def keypoints_convert(kpts, mode):
    """tools/mpii_coco_h36m.py: (T,J_in,2) -> ((T,17|19,2), valid mask (T,) int32)."""
    k = _cuda_f32(kpts, 'keypoints_convert')
    if k.dim() != 3 or k.shape[-1] != 2:
        raise GastError('keypoints_convert: (T,J,2) expected')
    T, Jin = int(k.shape[0]), int(k.shape[1])
    Jo = 19 if mode == KPT_COCO_H36M_TOE else 17
    out = torch.empty((T, Jo, 2), dtype=torch.float32, device=k.device)
    valid = torch.empty((T,), dtype=torch.int32, device=k.device)
    with torch.cuda.device(k.device):
        _check(L.load().gast_keypoints_convert(_p(k), _p(out), _p(valid), T, Jin, int(mode), C.c_void_p(_stream(k.device))),
               'gast_keypoints_convert')
    return out, valid


def normalize_screen(x, w, h, inverse=False):
    """common/camera.py:8-19 on (...,2) points."""
    x = _cuda_f32(x, 'normalize_screen')
    assert x.shape[-1] == 2
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _check(L.load().gast_normalize_screen(_p(x), _p(out), x.numel() // 2, float(w), float(h), 1 if inverse else 0,
                                              C.c_void_p(_stream(x.device))), 'gast_normalize_screen')
    return out


def camera_to_world(x, R, t=0):
    """common/camera.py:27-28 with one quaternion R (4,) and translation t (3,) or scalar for all points."""
    x = _cuda_f32(x, 'camera_to_world')
    assert x.shape[-1] == 3
    q = (C.c_float * 4)(*[float(v) for v in np.asarray(R, dtype=np.float32).reshape(4)])
    tv = np.broadcast_to(np.asarray(t, dtype=np.float32), (3,))
    tt = (C.c_float * 3)(*[float(v) for v in tv])
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _check(L.load().gast_camera_to_world(_p(x), _p(out), x.numel() // 3, q, tt, C.c_void_p(_stream(x.device))),
               'gast_camera_to_world')
    return out


# ------------------------------------------------------------------------------------------------
# The video demo's keypoint repair and placement of the lifted persons (tools/preprocess.py)
# ------------------------------------------------------------------------------------------------
_PREP_WS = {}


def _prep_ws(dev, nbytes):
    """scratch for the placement minima, grown on demand and kept per device"""
    ws = _PREP_WS.get(dev)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)
        _PREP_WS[dev] = ws
    return ws


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
    with torch.cuda.device(dev):
        _check(L.load().gast_h36m_coco_format(_p(k), _p(s), P, T, _p(out), _p(sout), _p(valid), _p(keep),
                                              C.c_void_p(_stream(dev))), 'gast_h36m_coco_format')
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
    with torch.cuda.device(k.device):
        _check(L.load().gast_revise_kpts(_p(k), _p(s), _p(v), P, T, J, _p(out), C.c_void_p(_stream(k.device))),
               'gast_revise_kpts')
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
    lib = L.load()
    wb = int(lib.gast_revise_skes_workspace_bytes(P, T))
    with torch.cuda.device(dev):
        ws = _prep_ws(dev, wb)
        _check(lib.gast_revise_skes(_p(pr), _p(fr), off.ctypes.data_as(C.POINTER(C.c_int64)), P, T, J, D, _p(k), _p(out),
                                    _p(ws), ws.numel(), C.c_void_p(_stream(dev))), 'gast_revise_skes')
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
    lib = L.load()
    wb = int(lib.gast_revise_skes_real_time_workspace_bytes(M))
    with torch.cuda.device(dev):
        ws = _prep_ws(dev, wb)
        _check(lib.gast_revise_skes_real_time(_p(pr), _p(k), M, J, D, float(width), _p(out), _p(ws), ws.numel(),
                                              C.c_void_p(_stream(dev))), 'gast_revise_skes_real_time')
    return out


# ------------------------------------------------------------------------------------------------
# N2: losses and the optimiser step
# ------------------------------------------------------------------------------------------------
_WS = {}


def _mpjpe_ws(dev):
    ws = _WS.get(dev)
    if ws is None:
        ws = torch.empty(int(L.load().gast_mpjpe_workspace_bytes()), dtype=torch.uint8, device=dev)
        _WS[dev] = ws
    return ws


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
        with torch.cuda.device(p.device):
            _check(L.load().gast_mpjpe(_p(p), _p(t), p.numel() // D, D, _p(loss), _p(dp), 1.0, _p(_mpjpe_ws(p.device)),
                                       C.c_void_p(_stream(p.device))), 'gast_mpjpe')
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
    with torch.cuda.device(p.device):
        _check(L.load().gast_p_mpjpe(_p(p), _p(t), N, J, _p(out), C.c_void_p(_stream(p.device))), 'gast_p_mpjpe')
    return out


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
        with torch.cuda.device(dev):
            _check(L.load().gast_adam_step(_p(self._table), int(self._table.shape[0]), _p(self.exp_avg), _p(self.exp_avg_sq),
                                           _p(self.max_exp_avg_sq), float(g['lr']), float(g['betas'][0]),
                                           float(g['betas'][1]), float(g['eps']), float(g['weight_decay']),
                                           self.step_count, C.c_void_p(_stream(dev))), 'gast_adam_step')
        # the kernel writes the parameters through raw pointers: bump their version counters so that everything
        # keyed on (data_ptr, _version) -- the engine's folded eval-mode constants -- sees the update
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
