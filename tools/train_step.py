"""GPU diagnostic: N training steps of BASELINE configs[2] (Optimized1f [3,3,3]/128ch, b = 128, dropout 0.05, FusedAdam
amsgrad) -- run under `ncu --metrics gpu__time_duration.sum` for the per-kernel device time of a step, or alone for the
wall time per step.

`train_step.py N eval`: the same model in eval() mode, forward + backward of an mpjpe loss (CUDA events over N
iterations after warm-up): with every parameter gradient and dL/dx, and input-only (parameters frozen); then the eval
forward alone under no_grad, and gast_eval_backward_workspace_bytes at b = 128 and 4096."""
import os
import sys
import time
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
from gast_b200 import synth  # noqa: E402
from gast_b200.trainer import DataParallelTrainer  # noqa: E402
from gast_b200.pipeline import FusedAdam  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f  # noqa: E402


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    J, b = 17, 128
    adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))
    m = SpatioTemporalModelOptimized1f(adj, J, 2, J, [3, 3, 3], channels=128, dropout=0.05)
    synth.randomize_module(m, 1)
    m = m.cuda()
    if len(sys.argv) > 2 and sys.argv[2] == 'eval':
        return eval_grad(m, steps, J, b)
    graphed = len(sys.argv) > 2 and sys.argv[2] == 'graph'
    if graphed:
        from gast_b200.trainer import GraphedTrainer
        tr = GraphedTrainer(m, lambda ps: FusedAdam(ps, lr=1e-3, amsgrad=True), (b, 27, J, 2), (b, 1, J, 3))
    else:
        tr = DataParallelTrainer(m, lambda ps: FusedAdam(ps, lr=1e-3, amsgrad=True))
    x = torch.from_numpy(synth.synth_input(b, 27, J, 2, seed=3)).cuda()
    y = torch.from_numpy(synth.synth_target(b, J, seed=4)).cuda()
    for _ in range(3):
        tr.step(x, y)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = tr.step(x, y)
    e1.record()
    t_issue = time.perf_counter() - t0
    torch.cuda.synchronize()
    print(('graphed ' if graphed else 'eager ') + 'steps %d: %.3f ms/step on the device stream, %.3f ms/step of host time to enqueue, loss %.5f'
          % (steps, e0.elapsed_time(e1) / steps, 1e3 * t_issue / steps, float(loss)))


def eval_grad(m, steps, J, b):
    m.eval()
    x = torch.from_numpy(synth.synth_input(b, 27, J, 2, seed=3)).cuda()
    y = torch.from_numpy(synth.synth_target(b, J, seed=4)).cuda()

    def fwd_bwd():
        xx = x.clone().requires_grad_()
        torch.mean(torch.norm(m(xx) - y, dim=3)).backward()

    def fwd():
        with torch.no_grad():
            m(x)

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    dev = torch.cuda.get_device_properties(0).name
    both = timed(fwd_bwd)
    m.requires_grad_(False)
    x_only = timed(fwd_bwd)
    m.requires_grad_(True)
    f = timed(fwd)
    h = list(m.__dict__['_gast_handles'].values())[0]
    ws = [int(h.lib.gast_eval_backward_workspace_bytes(h.h, n, 27, 1)) for n in (128, 4096)]
    print('%s, eval() b=%d 27f/128ch: forward+backward with parameter gradients and dx %.3f ms, input-only (dx) %.3f ms, '
          'forward alone (no_grad) %.3f ms; gast_eval_backward_workspace_bytes b=128: %d (%.1f MiB), b=4096: %d (%.2f GiB)'
          % (dev, b, both, x_only, f, ws[0], ws[0] / 2 ** 20, ws[1], ws[1] / 2 ** 30))


if __name__ == '__main__':
    main()
