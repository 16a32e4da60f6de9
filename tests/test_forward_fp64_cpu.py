"""Anchors the fp64 references of tests/test_gpu_forward_fp64.py.  CPU only.

  * The torch port (oracle/gast_torch_ref.py), in fp32 and in fp64, against goldens of the unmodified reference for
    the sub-module variants the GPU test sweeps: MultiGlobalGraph with 1 and 3 heads at J = 17, 19, 24, and
    SemCHGraphConv / SemGraphConv with out_features != in_features (tests/golden/make_golden.py:variant_cases).
  * The numpy oracle (oracle/gast_oracle.py) against the same goldens, and against the fp64 port on the model
    geometries the GPU test adds (one stage, five stages, a 5-wide first filter, dense, causal strided).
  * The 28- and 32-joint skeletons: the masks fp64ref restates equal the ones LocalGraph builds from its table entry,
    and fit the library's limits (J <= 32, at most 160 nonzeros per mask).
"""
import numpy as np
import pytest
import torch

from conftest import load_golden, golden_names
from gast_b200 import synth
from oracle import gast_oracle as O
from oracle import gast_torch_ref as TR
import fp64ref as R

TOL = 2e-5      # fp32 against fp32 in another operation order (as tests/test_oracle_golden.py)
VARIANTS = golden_names('var_')


def _params(meta, dtype):
    return {k: torch.from_numpy(v).to(dtype)
            for k, v in synth.synth_state([(k, tuple(s)) for k, s in meta['keys']], meta['seed']).items()}


def _port(g, dtype):
    meta = g['meta']
    p = _params(meta, dtype)
    x = torch.from_numpy(g['x']).to(dtype)
    with torch.no_grad():
        if meta['kind'] == 'mglobal':
            return TR.multi_global_graph(x, p, '')
        return TR.semch(x, p['W'], p['e'], torch.from_numpy(g['mask']), p.get('bias'))


def test_variant_goldens_cover_the_sweep():
    heads = {load_golden(n)['meta']['heads'] for n in VARIANTS if n.startswith('var_mglobal')}
    couts = {load_golden(n)['meta']['Cout'] for n in VARIANTS if not n.startswith('var_mglobal')}
    assert heads == {1, 3} and couts == {4, 36, 64, 200}


@pytest.mark.parametrize('name', VARIANTS)
def test_torch_port_matches_variant_golden(name):
    g = load_golden(name)
    y32 = _port(g, torch.float32).numpy()
    y64 = _port(g, torch.float64)
    assert y32.shape == g['y'].shape
    assert np.abs(y32 - g['y']).max() < TOL
    # the golden carries the reference's own fp32 rounding: fp64 sits within it
    assert np.abs(y64.numpy() - g['y']).max() < TOL * max(1.0, np.abs(g['y']).max())
    mx, l2 = R.errors(y32, y64)
    assert mx < 2e-6 and l2 < 2e-6, (mx, l2)


@pytest.mark.parametrize('name', VARIANTS)
def test_numpy_oracle_matches_variant_golden(name):
    g = load_golden(name)
    meta = g['meta']
    p = {k: v.numpy() for k, v in _params(meta, torch.float32).items()}
    if meta['kind'] == 'mglobal':
        y = O.multi_global_graph(g['x'], p, '')
    else:
        if meta['J'] in (17, 19):
            assert (O.local_masks(O.adj_from_parents(synth.skeleton_parents(meta['J'])))[1] == g['mask']).all()
        y = O.semch_graph_conv(g['x'], p['W'], p['e'], g['mask'], bias=p.get('bias'))
    assert np.abs(y - g['y']).max() < TOL


# (J, filter widths, channels, B, T, strided, causal, dense): model geometries of the GPU test at widths the numpy
# oracle finishes in seconds
GEOMETRIES = [
    (17, [3], 16, 3, 7, False, False, False),
    (17, [3], 8, 4, 3, True, False, False),
    (15, [3, 3, 3, 3, 3], 8, 1, 245, False, False, False),
    (16, [5, 3], 8, 2, 19, False, True, False),
    (19, [5, 3], 8, 3, 15, True, True, False),
    (16, [3, 3, 3], 8, 2, 30, False, False, True),
    (19, [3, 3, 3], 8, 2, 27, True, True, False),
]


@pytest.mark.parametrize('J,fw,ch,B,T,strided,causal,dense', GEOMETRIES)
def test_numpy_oracle_matches_fp64_port_on_new_geometries(J, fw, ch, B, T, strided, causal, dense):
    from model.gast_net import SpatioTemporalModel, SpatioTemporalModelOptimized1f
    if strided:
        m = SpatioTemporalModelOptimized1f(R.adj(J), J, 2, J, fw, causal=causal, channels=ch)
    else:
        m = SpatioTemporalModel(R.adj(J), J, 2, J, fw, causal=causal, channels=ch, dense=dense)
    synth.randomize_module(m, 13)
    x = synth.synth_input(B, T, J, 2, seed=17)
    y64 = R.model_forward64(m.state_dict(), x, J, fw, causal, strided, dense)
    p = {k: v.numpy() for k, v in m.state_dict().items()}
    yo = O.forward(x, p, O.adj_from_parents(synth.skeleton_parents(J)), fw, causal=causal, strided=strided, dense=dense)
    with torch.no_grad():
        y32 = TR.forward(torch.from_numpy(x), {k: v.clone() for k, v in m.state_dict().items()}, R.masks(J), fw,
                         causal=causal, strided=strided, dense=dense).numpy()
    assert yo.shape == tuple(y64.shape) == y32.shape
    for y in (yo, y32):
        mx, l2 = R.errors(y, y64)
        assert mx < 2e-6 and l2 < 2e-6, (mx, l2)


@pytest.mark.parametrize('J', [28, 32])
def test_many_joint_skeleton_masks(J, monkeypatch):
    from model.local_attention import LocalGraph
    R.install_tables(monkeypatch, J)
    lg = LocalGraph(R.adj(J), 8, 8)
    sym, con = R.masks(J)
    assert torch.equal(lg.gcn_sym.m, sym) and torch.equal(lg.gcn_con.m, con)
    assert torch.equal(sym, sym.T) and bool(torch.diagonal(con).all())
    assert 128 // J == 4 and int(sym.sum()) <= 160 and int(con.sum()) <= 160, (int(sym.sum()), int(con.sum()))
    distal, left, right = R.joint_table(J)
    assert len(left) == len(right) and not set(left) & set(right) and len(distal) == 7
    assert R.skeleton(J).num_joints() == J
