"""Device-side counterpart of the reference's common/camera.py (same names and signatures; under `device.` so that the
reference module is not shadowed): `normalize_screen_coordinates` (:8-12), `image_coordinates` (:15-19),
`world_to_camera` (:22-24), `camera_to_world` (:27-28, one quaternion for all points as reconstruction.py:204 /
gen_skes.py use it) and `project_to_2d` (:31-62, differentiable with respect to X).  numpy in -> numpy out (through
the device), CUDA tensor in -> CUDA tensor out."""
import numpy as np
import torch

from gast_b200 import pipeline as _P
from gast_b200.engine import GastError


def _run(fn, X):
    if isinstance(X, torch.Tensor):
        return fn(X)
    return fn(torch.as_tensor(np.ascontiguousarray(X, dtype=np.float32)).cuda()).cpu().numpy()


def normalize_screen_coordinates(X, w, h):
    assert X.shape[-1] == 2
    return _run(lambda x: _P.normalize_screen(x, w, h), X)


def image_coordinates(X, w, h):
    assert X.shape[-1] == 2
    return _run(lambda x: _P.normalize_screen(x, w, h, inverse=True), X)


def world_to_camera(X, R, t):
    assert X.shape[-1] == 3
    return _run(lambda x: _P.world_to_camera(x, R, t), X)


def camera_to_world(X, R, t):
    assert X.shape[-1] == 3
    return _run(lambda x: _P.camera_to_world(x, R, t), X)


class _ProjectFn(torch.autograd.Function):
    """project_to_2d of the points x with intrinsics row s for the points seg[s] .. seg[s+1]-1; d/dx on the device"""

    @staticmethod
    def forward(ctx, x, seg, intr):
        ctx.save_for_backward(x, seg, intr)
        return _P.project_to_2d_segments(x, seg, intr)

    @staticmethod
    def backward(ctx, g):
        x, seg, intr = ctx.saved_tensors
        return _P.project_to_2d_segments(x, seg, intr, grad_out=g.contiguous()), None, None


def project_to_2d(X, camera_params):
    """Project 3D points in camera space X (N, *, 3) with the intrinsics camera_params (N, 9) of each of the N rows
    (focal length 2, centre 2, radial distortion 3, tangential distortion 2).  Differentiable with respect to X; the
    intrinsics get no gradient and are refused when they require one."""
    assert X.shape[-1] == 3
    assert len(camera_params.shape) == 2
    assert camera_params.shape[-1] == 9
    assert X.shape[0] == camera_params.shape[0]
    if isinstance(camera_params, torch.Tensor) and camera_params.requires_grad:
        raise GastError('project_to_2d: no gradient with respect to the intrinsics; pass them detached')

    def run(x):
        x = x.contiguous()
        N = int(x.shape[0])
        intr = torch.as_tensor(camera_params, dtype=torch.float32).to(x.device).contiguous()
        seg = torch.arange(N + 1, dtype=torch.int64, device=x.device) * (x.numel() // (3 * N) if N else 0)
        return _ProjectFn.apply(x, seg, intr)

    return _run(run, X)
