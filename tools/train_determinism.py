"""GPU diagnostic: run-to-run determinism of the training gradients (same weights, same batch, two runs) and the
fraction of parameter entries that differ after three Adam(amsgrad) steps between two identically-seeded trainers
(eager vs eager, eager vs CUDA graph), on one GEMM core.

    python tools/train_determinism.py [channels] [core]     core: 0 = tensor cores where possible (default), 1 = FFMA"""
import os
import sys
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'gast-net-3dposeestimation_b200'))
sys.path.insert(0, REPO)
from gast_b200 import engine, synth  # noqa: E402
from gast_b200.trainer import DataParallelTrainer, GraphedTrainer  # noqa: E402
from gast_b200.pipeline import FusedAdam  # noqa: E402
from common.skeleton import Skeleton  # noqa: E402
from common.graph_utils import adj_mx_from_skeleton  # noqa: E402
from model.gast_net import SpatioTemporalModelOptimized1f  # noqa: E402

J = 17
adj = adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))


def make(ch):
    m = SpatioTemporalModelOptimized1f(adj, J, 2, J, [3, 3, 3], dropout=0.0, channels=ch)
    synth.randomize_module(m, 3)
    return m.cuda()


def grads_once(m, x, y):
    m.train()
    for p in m.parameters():
        p.grad = None
    out = m(x)
    loss = torch.mean(torch.norm(out - y, dim=3))
    loss.backward()
    return {k: p.grad.detach().clone() for k, p in m.named_parameters()}, float(loss)


def tc_launches(m):
    """tensor-core GEMM launches the model's handle has counted (0 when every training GEMM ran on FFMA)"""
    h = list(m.__dict__['_gast_handles'].values())[0]
    return int(h.lib.gast_last_tc_launch_count(h.h))


def main():
    ch = int(sys.argv[1]) if len(sys.argv) > 1 else 32
    core = int(sys.argv[2]) if len(sys.argv) > 2 else 0
    engine.set_gemm_core(core)
    B = 16
    print('gemm core %d channels=%d' % (core, ch))
    x = torch.from_numpy(synth.synth_input(B, 27, J, 2, seed=40)).cuda()
    y = torch.from_numpy(synth.synth_target(B, J, seed=50)).cuda()
    m = make(ch)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    g1, l1 = grads_once(m, x, y)
    print('tensor-core GEMM launches in the first training step: %d' % tc_launches(m))
    m.load_state_dict(sd)
    g2, l2 = grads_once(m, x, y)
    nd = [(k, float((g1[k] - g2[k]).abs().max()), float(g1[k].abs().max())) for k in g1 if not torch.equal(g1[k], g2[k])]
    print('run-to-run: loss %.9g vs %.9g; %d of %d gradient tensors differ bitwise' % (l1, l2, len(nd), len(g1)))
    for k, d, s in sorted(nd, key=lambda t: -t[1] / max(t[2], 1e-30))[:12]:
        print('   %-70s max|d| %.3e  max|g| %.3e' % (k, d, s))
    opt = lambda ps: FusedAdam(ps, lr=1e-3, amsgrad=True)  # noqa: E731
    xs = [torch.from_numpy(synth.synth_input(B, 27, J, 2, seed=40 + i)).cuda() for i in range(3)]
    ys = [torch.from_numpy(synth.synth_target(B, J, seed=50 + i)).cuda() for i in range(3)]

    def frac(a, b):
        bad = tot = 0
        for (k, p), (_, q) in zip(a.model.named_parameters(), b.model.named_parameters()):
            if k == 'init_bn.bias':
                continue
            bad += int(((p - q).abs() > 1e-5).sum())
            tot += p.numel()
        return bad, tot
    a = DataParallelTrainer(make(ch), opt)
    b = DataParallelTrainer(make(ch), opt)
    c = GraphedTrainer(make(ch), opt, (B, 27, J, 2), (B, 1, J, 3))
    c.model.load_state_dict(a.model.state_dict())
    for xx, yy in zip(xs, ys):
        la, lb, lc = a.step(xx, yy), b.step(xx, yy), c.step(xx, yy)
        print('   step losses eager %.9g eager %.9g graph %.9g' % (float(la), float(lb), float(lc)))
    print('after 3 steps: eager vs eager differ in %d of %d entries; eager vs graph in %d of %d' % (frac(a, b) + frac(a, c)))


if __name__ == '__main__':
    main()
