"""The numpy restatement of the library's dropout masks (tests/dropoutref.py) on the CPU: the hash against a
pure-Python-int restatement of dropout_mask_kernel (csrc/train_kernels.cuh), the keep rate, the independence of the
masks of different sites and graph replays, and the port's mask injection (oracle/gast_torch_ref.py, `drop=`)."""
import numpy as np
import pytest
import torch

from conftest import load_golden, golden_names
import dropoutref as D
import kinkfree as K

U64 = (1 << 64) - 1


def _kernel_keep(seed, k, i, p, dstate):
    """dropout_mask_kernel for element i of site k, in Python ints: (x, keep)"""
    s = (seed + 0x51ED270B * k + dstate) & U64
    x = (i * 0x9E3779B97F4A7C15 + s) & U64
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & U64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & U64
    x ^= x >> 31
    u = np.float32(x >> 40) * np.float32(1.0 / 16777216.0)
    return x, int(u >= np.float32(p))


def _sigma5(n, q):
    return 5.0 * (n * q * (1.0 - q)) ** 0.5


def test_hash_matches_the_kernel_formula():
    idx = [0, 1, 2, 255, 256, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 12345, 3 * 2 ** 33 + 7, 2 ** 40 + 1,
           2 ** 62 + 5]
    for seed in (0, 1, D.engine_seed(K.DROP_SEED), 2 ** 62 - 1):
        for k in (1, 2, 8, 11, 64):
            for dstate in (0, D.DSTATE_STEP, (3 * D.DSTATE_STEP) & U64, U64):
                for p in (0.05, 0.25, 0.5, 0.9):
                    x = D.bits(seed, k, np.array(idx, np.uint64), dstate)
                    got = (D.uniform(x) >= np.float32(p)).astype(np.uint8)
                    for j, i in enumerate(idx):
                        xr, kr = _kernel_keep(seed, k, i, p, dstate)
                        assert int(x[j]) == xr and int(got[j]) == kr, (seed, k, dstate, i)
    # keep() is the same hash over 0..n-1
    n = 1000
    ref = [_kernel_keep(7, 3, i, 0.25, D.DSTATE_STEP)[1] for i in range(n)]
    assert D.keep(7, 3, n, 0.25, D.DSTATE_STEP).tolist() == ref


def test_scale_and_engine_seed():
    for p in (0.05, 0.25, 0.5, 0.9):
        s = D.scale(p)
        assert s.dtype == np.float32 and s == np.float32(1) / (np.float32(1) - np.float32(p))
    assert D.scale(0.9) == np.float32(1) / np.float32(np.float32(1) - np.float32(0.9))   # ~10, not 10.000000000000002
    for S in (0, K.DROP_SEED, 12345):
        torch.manual_seed(S)
        assert D.engine_seed(S) == int(torch.randint(0, 2 ** 62, (1,)).item())


@pytest.mark.parametrize('p', [0.05, 0.25, 0.5, 0.9])
def test_keep_fraction(p):
    """over 2^22 draws, within 5 sigma of the exact rate: u lives on the 2^-24 grid and the threshold is float32(p)"""
    n = 1 << 22
    q = (2 ** 24 - int(np.ceil(np.float64(np.float32(p)) * 2 ** 24))) / 2 ** 24
    kept = int(D.keep(D.engine_seed(K.DROP_SEED), 1, n, p).sum())
    assert abs(kept - n * q) <= _sigma5(n, q), (kept, n * q)


@pytest.mark.parametrize('p', [0.05, 0.5])
def test_sites_and_replays_draw_independent_masks(p):
    """the masks of different sites and of different graph counters agree at the independent-coin rate"""
    n = 1 << 20
    seed = D.engine_seed(K.DROP_SEED)
    q = float(D.keep(seed, 1, n, p).mean())
    agree = q * q + (1 - q) * (1 - q)
    pairs = [((1, 0), (2, 0)), ((1, 0), (4, 0)), ((1, 0), (1, D.DSTATE_STEP)), ((2, D.DSTATE_STEP), (3, 0)),
             ((5, (7 * D.DSTATE_STEP) & U64), (5, (8 * D.DSTATE_STEP) & U64))]
    for (ka, da), (kb, db) in pairs:
        same = int((D.keep(seed, ka, n, p, da) == D.keep(seed, kb, n, p, db)).sum())
        assert abs(same - n * agree) <= _sigma5(n, agree), ((ka, da), (kb, db), same / n, agree)


def test_streams_of_sites_and_replays_never_overlap():
    """every (site <= 64, replay <= 4096) stream is the hash of i * gamma + s; two such streams are the same sequence
    shifted by d = (s2 - s1) / gamma (mod 2^64), and every such shift is beyond 2^40 elements either way"""
    dk = np.arange(-63, 64, dtype=np.int64)
    dr = np.arange(-4096, 4097, dtype=np.int64)
    with np.errstate(over='ignore'):
        delta = (dk[:, None].astype(np.uint64) * np.uint64(D.SITE_MUL)
                 + dr[None, :].astype(np.uint64) * np.uint64(D.DSTATE_STEP))
        d = delta * np.uint64(pow(D.GOLDEN_GAMMA, -1, 1 << 64))
        back = np.uint64(0) - d
    d[63, 4096] = back[63, 4096] = np.uint64(U64)        # the stream against itself
    assert int(np.minimum(d, back).min()) > 2 ** 40


def test_site_order_and_shapes():
    assert D.sites(3) == ['layers_graph_conv.0.local_graph_layer.cat_bn.', 'layers_graph_conv.0.global_graph_layer.cat_bn.',
                          'layers_bn.1.', 'layers_graph_conv.1.local_graph_layer.cat_bn.',
                          'layers_graph_conv.1.global_graph_layer.cat_bn.',
                          'layers_bn.3.', 'layers_graph_conv.2.local_graph_layer.cat_bn.',
                          'layers_graph_conv.2.global_graph_layer.cat_bn.']
    for L in (2, 3, 4):
        assert len(D.sites(L)) == 3 * L - 1


def _site_run(case, drop):
    """the port's train forward of `case` in fp64 at its synthetic weights with `drop`; every site's ReLU input and
    dropout output, in call order"""
    from oracle import gast_torch_ref as TR
    sd = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in K.module(case).state_dict().items()}
    relu_in, out = {}, []

    def tap(name, h):
        relu_in[name] = h.detach().clone()

    def rec(name, h):
        r = drop(name, h) if callable(drop) else h
        out.append((name, h.detach().clone(), r.detach().clone()))
        return r
    with torch.no_grad():
        y = TR.forward(K.inputs(case).double(), sd, K.masks(case.J), case.fw, causal=case.causal, strided=case.strided,
                       dense=case.dense, training=True, drop=rec, tap=tap)
    return y, relu_in, out


@pytest.mark.parametrize('name', ['o1f_j19_c160_train_drop50', 'causal_T40_j17_c48_train_drop25',
                                  'dense_j15_c16_train_drop05', 'o1f_j17_c32_3333_train_drop05'])
def test_port_applies_the_masks_at_every_site(name):
    case = K.CASES[name]
    masks = K.drop_masks(case)
    assert list(masks) == D.sites(len(case.fw))
    # all-ones masks change no bit of the port's train forward without dropout
    from oracle import gast_torch_ref as TR
    sd = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in K.module(case).state_dict().items()}
    x = K.inputs(case).double()
    ones = D.dropper({k: torch.ones_like(v) for k, v in masks.items()})
    kw = dict(causal=case.causal, strided=case.strided, dense=case.dense, training=True)
    with torch.no_grad():
        y0 = TR.forward(x, sd, K.masks(case.J), case.fw, drop=0.0, **kw)
        y1 = TR.forward(x, sd, K.masks(case.J), case.fw, drop=ones, **kw)
    assert torch.equal(y0, y1)
    # with the masks: each site's output is mask * scale * relu(bn(...)), in site order, on the site's whole output
    _, relu_in, out = _site_run(case, D.dropper(masks))
    assert [n for n, _, _ in out] == D.sites(len(case.fw))
    s = float(D.scale(case.drop))
    for site, (n, h, r) in zip(D.sites(len(case.fw)), out):
        assert torch.equal(h, torch.relu(relu_in[site])), site
        keep = masks[site] != 0
        assert torch.equal(r, torch.where(keep, h * s, torch.zeros_like(h))), site
        frac = float(keep.double().mean())
        assert abs(frac - (1 - case.drop)) < 0.05, (site, frac)
    # the mask is the emulator's keep() over the site's output in (b, t, j, c) order
    seed = D.engine_seed(K.DROP_SEED)
    for k, (site, m) in enumerate(masks.items()):
        flat = (m.permute(0, 2, 3, 1).reshape(-1) != 0).numpy().astype(np.uint8)
        assert np.array_equal(flat, D.keep(seed, k + 1, flat.size, case.drop)), site


def test_eval_mode_ignores_the_masks():
    case = K.CASES['o1f_j19_c160_eval']
    from oracle import gast_torch_ref as TR
    sd = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in K.module(case).state_dict().items()}
    called = []
    with torch.no_grad():
        y0 = TR.forward(K.inputs(case).double(), sd, K.masks(case.J), case.fw, strided=True)
        y1 = TR.forward(K.inputs(case).double(), sd, K.masks(case.J), case.fw, strided=True,
                        drop=lambda n, h: called.append(n))
    assert torch.equal(y0, y1) and not called


@pytest.mark.parametrize('name', [n for n in golden_names('grad_') if 'drop' in n])
def test_golden_masks_are_the_emulators(name):
    """the masks a dropout golden stores are those the library draws after torch.manual_seed(meta['drop_seed'])"""
    g = load_golden(name)
    meta = g['meta']
    got = D.golden_masks(g)
    ref = D.masks(meta, meta['B'], meta['T'], meta['J'], meta['dropout'], D.engine_seed(meta['drop_seed']))
    assert list(got) == list(ref) == D.sites(len(meta['filter_widths']))
    for k in ref:
        assert torch.equal(got[k], ref[k]), k
