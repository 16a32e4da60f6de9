"""CPU checks of the boundary: the C-ABI library loads and exports every symbol that
include/gast_b200.h declares, the header declares every extern "C" definition under csrc/, and the
ctypes bindings are those its prototypes state; the drop-in modules keep the reference's API surface; and the
product path refuses to run without a GPU (no fallback)."""
import ctypes as C
import os
import re
import pytest
import torch
from conftest import REPO, load_golden, golden_names
from gast_b200 import _lib, synth


def _adj(J):
    from common.skeleton import Skeleton
    from common.graph_utils import adj_mx_from_skeleton
    return adj_mx_from_skeleton(Skeleton(synth.skeleton_parents(J), [], []))


def _uncommented(path):
    return re.sub(r'/\*.*?\*/|//[^\n]*', '', open(path).read(), flags=re.S)


def test_library_exports_every_declared_symbol():
    hdr = _uncommented(os.path.join(REPO, 'include', 'gast_b200.h'))
    declared = set(re.findall(r'\b(gast_[a-z_0-9]+)\s*\(', hdr))
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    lib = _lib.load()
    for s in declared:
        assert getattr(lib, s) is not None
    assert b'sm_90a' in lib.gast_version()


def test_header_declares_every_extern_c_definition():
    csrc = os.path.join(REPO, 'gast-net-3dposeestimation_b200', 'csrc')
    defined = []
    for f in sorted(os.listdir(csrc)):
        if f.endswith(('.cu', '.cuh')):
            defined += re.findall(r'extern\s+"C"\s+[\w\s*]*?\b(gast_\w+)\s*\(', _uncommented(os.path.join(csrc, f)))
    assert defined and len(defined) == len(set(defined)) and len(_lib.SYMBOLS) == len(set(_lib.SYMBOLS))
    assert set(defined) == set(_lib.SYMBOLS), set(defined) ^ set(_lib.SYMBOLS)


def test_bindings_derived_from_the_header():
    lib = _lib.load()
    train = lib.gast_forward_train.argtypes
    assert len(train) == 10 and train[6] is C.c_uint64 and train[5] is C.c_float and train[0] is C.c_void_p
    assert lib.gast_last_error.restype is C.c_char_p and lib.gast_version.restype is C.c_char_p
    assert lib.gast_destroy.restype is None
    assert lib.gast_adam_chunk.argtypes == [] and lib.gast_adam_chunk.restype is C.c_int32
    assert lib.gast_debug_set_gemm_audit.argtypes == [C.c_void_p] * 3            # a callback typedef is a pointer
    assert lib.gast_bind.argtypes == [C.c_void_p, C.c_int32] + [C.c_void_p] * 3
    assert lib.gast_workspace_bytes.restype is C.c_size_t


def test_prototype_parser():
    hdr = '''#define X 1
    typedef int (*gast_cb_fn)(int32_t phase, void* user);   /* a comment: int gast_ghost(int); */
    typedef struct gast_s { const float* p; int32_t n; } gast_s;
    int gast_a(const gast_s* const* s, int64_t n, double w, gast_cb_fn fn, uint64_t seed);
    size_t gast_b(void);
    void gast_c(float x, int k, size_t n);
    const char* gast_d(void);'''
    assert _lib.prototypes(hdr) == [
        ('gast_a', C.c_int, [C.c_void_p, C.c_int64, C.c_double, C.c_void_p, C.c_uint64]),
        ('gast_b', C.c_size_t, []), ('gast_c', None, [C.c_float, C.c_int, C.c_size_t]), ('gast_d', C.c_char_p, [])]
    for bad in ('int gast_e(unsigned n);', 'int gast_e(long long n);', 'int gast_e(float q[4]);',
                'int gast_e(enum gast_kind k);', 'void* gast_e(void);', 'uint8_t gast_e(void);'):
        with pytest.raises(RuntimeError, match='gast_e'):
            _lib.prototypes(hdr + '\n' + bad)


def test_star_import_namespace_and_state_dict_keys():
    ns = {}
    exec('from model.gast_net import *', ns)
    for name in ('torch', 'nn', 'SpatioTemporalModel', 'SpatioTemporalModelOptimized1f',
                 'GraphAttentionBlock', 'LocalGraph', 'MultiGlobalGraph', 'SingleGlobalGraph'):
        assert name in ns, name        # trainval.py:60 needs `nn` through this star import
    import model.gast_net as G
    assert 'gast-net-3dposeestimation_b200' in G.__file__
    for name in golden_names('model_') + golden_names('cfg'):
        meta = load_golden(name)['meta']
        cls = G.SpatioTemporalModelOptimized1f if meta['strided'] else G.SpatioTemporalModel
        kw = {} if meta['strided'] else {'dense': meta['dense']}
        m = cls(_adj(meta['J']), meta['J'], 2, meta['J'], meta['filter_widths'], causal=meta['causal'],
                dropout=0.05, channels=meta['channels'], **kw)
        assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == meta['keys']
        assert m.pad == meta['pad'] and m.causal_shift == meta['causal_shift']
        assert m.receptive_field() == meta['receptive_field']
        assert m.total_causal_shift() == meta['total_causal_shift']


def test_adjacency_matches_reference_pattern():
    a = _adj(17)
    assert a.dtype == torch.float32 and a.shape == (17, 17)
    assert int((a > 0).sum()) == 49 and torch.allclose(a.sum(1), torch.ones(17))
    from model.local_attention import local_adjacencies
    s, c = local_adjacencies(a)
    assert int((s > 0).sum()) == 29 and int((c > 0).sum()) == 54
    g = load_golden('mod_semch_17_32')
    assert ((c > 0).numpy() == g['mask']).all()


def test_no_cpu_fallback():
    from model.gast_net import SpatioTemporalModel
    m = SpatioTemporalModel(_adj(17), 17, 2, 17, [3, 3, 3], channels=16).eval()
    with pytest.raises(RuntimeError, match='no CPU path'):
        m(torch.zeros(1, 27, 17, 2))
    with pytest.raises(AssertionError):
        m(torch.zeros(1, 27, 16, 2))


def test_skeleton_remove_joints_like_reference():
    from common.skeleton import Skeleton
    parents = [-1, 0, 1, 2, 3, 4, 0, 6, 7, 8, 9, 0, 11, 12, 13, 14, 12, 16, 17, 18, 19, 20, 19, 22, 12, 24,
               25, 26, 27, 28, 27, 30]
    sk = Skeleton(parents=list(parents), joints_left=[6, 7, 8, 9, 10, 16, 17, 18, 19, 20, 21, 22, 23],
                  joints_right=[1, 2, 3, 4, 5, 24, 25, 26, 27, 28, 29, 30, 31])
    sk.remove_joints([4, 5, 9, 10, 11, 16, 20, 21, 22, 23, 24, 28, 29, 30, 31])   # h36m_dataset.py:253
    got = [int(q) for q in sk.parents()]
    assert got == [-1, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 7, 11, 12, 7, 14, 15]   # same as the reference class
    got[11] = 8
    got[14] = 8                                   # shoulder rewiring, h36m_dataset.py:284-285
    assert got == synth.H36M_PARENTS_17
    assert sk.joints_left() == [4, 5, 6, 11, 12, 13] and sk.joints_right() == [1, 2, 3, 14, 15, 16]


def test_reference_checkpoint_layout_loads(tmp_path):
    """N4: a checkpoint in the reference's on-disk layout ({'model_pos': state_dict}, trainval.py:192-199),
    also with the `module.` prefixes an nn.DataParallel-wrapped model writes, loads strictly."""
    from model.gast_net import SpatioTemporalModel
    from gast_b200.checkpoint import load_checkpoint
    src = SpatioTemporalModel(_adj(17), 17, 2, 17, [3, 3, 3], channels=16)
    synth.randomize_module(src, 4)
    for prefix in ('', 'module.'):
        path = os.path.join(str(tmp_path), 'm%d.bin' % len(prefix))
        torch.save({'epoch': 3, 'lr': 1e-3, 'model_pos': {prefix + k: v for k, v in src.state_dict().items()}}, path)
        dst = SpatioTemporalModel(_adj(17), 17, 2, 17, [3, 3, 3], channels=16)
        chk = load_checkpoint(dst, path)
        assert chk['epoch'] == 3
        for (k, a), (_, b) in zip(src.state_dict().items(), dst.state_dict().items()):
            assert torch.equal(a, b), k
    plain = SpatioTemporalModel(_adj(17), 17, 2, 17, [3, 3, 3], channels=16)
    plain.load_state_dict(torch.load(path.replace('m7', 'm0'))['model_pos'])      # reconstruction.py:239-240 verbatim


def test_device_side_callers_have_no_cpu_path():
    """The device-side counterparts of the caller modules (device/) import without a GPU, keep the reference's
    names, and refuse CPU tensors instead of silently computing on the host."""
    import numpy as np
    import device.common.loss as L
    import device.common.camera as Cm
    import device.common.generators as Gn
    import device.tools.mpii_coco_h36m as K
    from gast_b200 import pipeline as P
    from gast_b200.stream import PipelinedLifter
    from model.gast_net import SpatioTemporalModel
    for mod, names in ((L, ('mpjpe', 'p_mpjpe')), (Cm, ('normalize_screen_coordinates', 'image_coordinates', 'camera_to_world')),
                       (Gn, ('ChunkedGenerator', 'UnchunkedGenerator')), (K, ('coco_h36m', 'mpii_h36m', 'coco_h36m_toe_format'))):
        for n in names:
            assert callable(getattr(mod, n)), n
    a = torch.zeros(4, 1, 17, 3)
    with pytest.raises(RuntimeError, match='no CPU path'):
        L.mpjpe(a, a)
    with pytest.raises(RuntimeError, match='no CPU path'):
        P.keypoints_convert(torch.zeros(3, 17, 2), P.KPT_COCO_H36M)
    with pytest.raises(RuntimeError, match='no CPU path'):
        PipelinedLifter(SpatioTemporalModel(_adj(17), 17, 2, 17, [3, 3, 3], channels=16))
    # the pair list and its shuffling are host logic shared with the oracle: identical to the reference's order
    from oracle import pipeline_oracle as PO
    pairs = PO.chunk_pairs((40, 7, 25), 1, True)
    assert pairs.shape == (144, 4) and pairs[:, 3].sum() == 72
    assert np.array_equal(pairs[:2], [[0, 0, 1, 0], [0, 1, 2, 0]]) and np.array_equal(pairs[40], [0, 0, 1, 1])
