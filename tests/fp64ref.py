"""fp64 references for the forward checks of tests/test_gpu_forward_fp64.py and tests/test_forward_fp64_cpu.py.

The reference is the torch-CPU port of the lifting path (oracle/gast_torch_ref.py) run in torch.float64.  It takes
the local masks explicitly, so it also serves skeletons that are not in the reference's joint tables: the 32-joint
Human3.6M skeleton (the raw one, h36m_dataset.py) and a 28-joint subset of it, whose tables are given here.

Errors are reported as two numbers against the fp64 output y64: max |y - y64| / max |y64| and the relative L2 error
|y - y64| / |y64|.
"""
import numpy as np
import torch

from gast_b200 import synth

# the raw 32-joint Human3.6M skeleton (parents, joints_left, joints_right), as common/skeleton.py is built for it
H36M32_PARENTS = [-1, 0, 1, 2, 3, 4, 0, 6, 7, 8, 9, 0, 11, 12, 13, 14, 12, 16, 17, 18, 19, 20, 19, 22, 12, 24, 25, 26,
                  27, 28, 27, 30]
H36M32_LEFT = [6, 7, 8, 9, 10, 16, 17, 18, 19, 20, 21, 22, 23]
H36M32_RIGHT = [1, 2, 3, 4, 5, 24, 25, 26, 27, 28, 29, 30, 31]
H36M28_REMOVED = [5, 10, 23, 31]      # one toe end per foot and one hand end per hand


def skeleton(J):
    """the common.skeleton.Skeleton of J joints: the reference's for J = 15, 16, 17, 19; for J = 32 the raw Human3.6M
    skeleton and for J = 28 that skeleton without H36M28_REMOVED (Skeleton.remove_joints re-parents the children)"""
    from common.skeleton import Skeleton
    if J in (15, 16, 17, 19):
        return Skeleton(synth.skeleton_parents(J), [], [])
    s = Skeleton(list(H36M32_PARENTS), list(H36M32_LEFT), list(H36M32_RIGHT))
    if J == 28:
        s.remove_joints(list(H36M28_REMOVED))
    assert s.num_joints() == J, J
    return s


def joint_table(J):
    """(distal, left, right) of model.local_attention._JOINT_TABLES for J = 28 / 32: the leaf joints are the distal
    ones"""
    s = skeleton(J)
    parents = [int(q) for q in s.parents()]
    return ([j for j in range(J) if j not in parents], [int(j) for j in s.joints_left()],
            [int(j) for j in s.joints_right()])


def install_tables(monkeypatch, J):
    """give model.local_attention._JOINT_TABLES an entry for J = 28 / 32 for the duration of a test"""
    import model.local_attention as LA
    if J not in LA._JOINT_TABLES:
        monkeypatch.setitem(LA._JOINT_TABLES, J, joint_table(J))


def adj(J):
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(skeleton(J))


def masks(J):
    """(sym, con) boolean masks of J joints as LocalGraph builds them (local_attention.py:92-114), restated here from
    the adjacency and joint_table so that it does not depend on the module's table"""
    a = adj(J).double().numpy()
    if J in (15, 16, 17, 19):
        from oracle import gast_oracle as O
        distal, left, right = O._TABLES[J]
    else:
        distal, left, right = joint_table(J)
    sym = np.eye(J, dtype=bool)
    for l, r in zip(left, right):
        sym[l, r] = sym[r, l] = True
    con = np.where(np.isin(np.arange(J), distal)[:, None], a @ a, a) > 0
    return torch.from_numpy(sym), torch.from_numpy(con)


def f64(sd):
    """a state_dict as float64 CPU tensors (integer buffers unchanged)"""
    return {k: (v.detach().cpu().double() if v.dtype.is_floating_point else v.detach().cpu()) for k, v in sd.items()}


def model_forward64(sd, x, J, fw, causal=False, strided=False, dense=False):
    """the eval-mode model forward in fp64 (gast_torch_ref.forward)"""
    from oracle import gast_torch_ref as TR
    with torch.no_grad():
        return TR.forward(torch.as_tensor(x).double(), f64(sd), masks(J), fw, causal=causal, strided=strided,
                          dense=dense)


def errors(y, y64):
    """(max |y - y64| / max |y64|, |y - y64| / |y64|)"""
    y = torch.as_tensor(y).double().cpu()
    y64 = torch.as_tensor(y64).double().cpu()
    assert y.shape == y64.shape, (tuple(y.shape), tuple(y64.shape))
    d = y - y64
    return float(d.abs().max() / y64.abs().max()), float(d.norm() / y64.norm())
