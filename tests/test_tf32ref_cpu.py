"""The TF32 restatement (tests/tf32ref.py) on the CPU.

- Rounding off, it reproduces the reference's goldens (model_*, cfg*, tc_*, mod_*) at fp32 rounding level: this pins
  the folded algebra (BN folded into the convs, [W0 | W1] SemCH GEMM, collapsed theta / phi, stacked `g`, 3-segment
  block GEMM, tap-gathered temporal GEMMs) to the reference.
- Rounding on, it moves the poses by TF32's amount.  Measured on these goldens' synthetic weights: max |dy| / max |y|
  between 3.5e-4 (a model with one rounded GEMM) and 2.7e-3, i.e. 2.2e-4 to 4.4e-3 absolute at |y| of 0.6-3.
- The rounding function matches cvt.rna.tf32.f32 bit for bit on hand-made cases.
"""
import numpy as np
import pytest

from conftest import load_golden, golden_names
from oracle import gast_oracle as O
from gast_b200 import synth
import tf32ref as R

TOL = 2e-5          # the fp32 reference against an fp64 restatement in another op order (test_oracle_golden.TOL)


def params(meta):
    return synth.synth_state([(k, tuple(s)) for k, s in meta['keys']], meta['seed'])


def masks_for(J):
    return O.local_masks(O.adj_from_parents(synth.skeleton_parents(J)))


def _model(name, rnd):
    g = load_golden(name)
    m = g['meta']
    y, gem = R.forward(g['x'], params(m), masks_for(m['J']), m['filter_widths'], causal=m['causal'],
                       strided=m['strided'], dense=m['dense'], rnd=rnd)
    return g, y, gem


MODELS = golden_names('model_') + golden_names('cfg') + golden_names('tc_')


@pytest.mark.parametrize('name', MODELS)
def test_unrounded_restatement_reproduces_reference_goldens(name):
    if name.startswith('cfg1'):
        pytest.skip('large dilated case (CPU time): its configuration is covered by cfg2 / cfg3')
    g, y, gem = _model(name, False)
    assert y.shape == g['y'].shape
    assert np.abs(y - g['y']).max() < TOL
    # the GEMM count of the device forward: 5 per block, 2 per temporal stage
    L = len(g['meta']['filter_widths'])
    assert gem.count == 5 * L + 2 * (L - 1)
    if name.startswith('tc_') or name.startswith('cfg'):
        assert gem.tc == gem.count          # widths that are multiples of 32: every GEMM on the tensor cores


@pytest.mark.parametrize('name', ['model_17_35_c8_full_T17', 'model_17_333_c16_1f_T27', 'cfg3_17_333_c128_1f_T27',
                                  'tc_17_333_c32_dense_T28', 'tc_17_33333_c32_1f_T243', 'tc_19_333_c32_1f_T27',
                                  'tc_17_3333_c64_causal_full_T90'])
def test_rounding_moves_poses_by_tf32s_amount(name):
    _, y0, _ = _model(name, False)
    _, y1, gem = _model(name, True)
    rel = np.abs(y1 - y0).max() / np.abs(y0).max()
    lo = 1e-4 if gem.tc == gem.count else 3e-5
    assert lo < rel < 5e-3, rel


def _module(name, kind, rnd):
    g = load_golden(name)
    m = g['meta']
    p = params(m)
    if kind in ('semch', 'semgc'):
        masks = g['mask'].astype(bool)
    else:
        masks = masks_for(m['J'])
    x = g['x'].transpose(0, 3, 1, 2) if kind == 'block' else g['x']      # block goldens keep x as (B, T, J, C)
    return g, R.module_forward(kind, x, p, masks, rnd=rnd)


MODULES = [('mod_block_17_32', 'block'), ('mod_block_19_16', 'block'), ('mod_local_17_32', 'local'),
           ('mod_mglobal_17_32', 'mglobal'), ('mod_global_17_32', 'global'), ('mod_semch_17_32', 'semch'),
           ('mod_semgc_17_32', 'semgc')]


@pytest.mark.parametrize('name,kind', MODULES)
def test_unrounded_modules_reproduce_reference_goldens(name, kind):
    g, (y, gem) = _module(name, kind, False)
    assert y.shape == g['y'].shape
    assert np.abs(y - g['y']).max() < TOL
    _, (y1, _) = _module(name, kind, True)
    rel = np.abs(y1 - y).max() / np.abs(y).max()
    if gem.tc:
        assert 1e-5 < rel < 5e-3, rel
    else:
        assert rel == 0.0


# ------------------------------------------------------------------------------------------------------------------
# the rounding function
# ------------------------------------------------------------------------------------------------------------------
def _bits(v):
    return np.asarray(v, np.float32).view(np.uint32)


def _f(u):
    return np.asarray(u, np.uint32).view(np.float32)


def test_tf32_rounding_bit_for_bit():
    # (input bits, expected bits): the low 13 bits are dropped, rounding to nearest with ties away from zero
    cases = [
        (0x3F800000, 0x3F800000),      # 1.0: exact
        (0x3F800FFF, 0x3F800000),      # just below half an ulp: down
        (0x3F801000, 0x3F802000),      # exactly half: away from zero (up)
        (0x3F803000, 0x3F804000),      # half above an odd tf32 mantissa: still away (not to even)
        (0x3F801001, 0x3F802000),      # above half: up
        (0xBF801000, 0xBF802000),      # negative tie: away from zero (more negative)
        (0xBF800FFF, 0xBF800000),      # negative below half: towards zero
        (0x3FFFF000, 0x40000000),      # 2 - 2^-11 (tie at the top of a binade): carries into the exponent, 2.0
        (0x3FFFEFFF, 0x3FFFE000),      # just below it: stays in [1, 2)
        (0xBFFFF000, 0xC0000000),      # negative: -2.0
        (0x7F7FFFFF, 0x7F800000),      # FLT_MAX: rounds past the largest tf32 to +inf
        (0x7F7FE000, 0x7F7FE000),      # largest tf32: exact
        (0x7F7FEFFF, 0x7F7FE000),      # below half an ulp under FLT_MAX range: stays finite
        (0x0DA24260, 0x0DA24000),      # ~1e-30: ordinary rounding at tiny magnitude
        (0x0DA25000, 0x0DA26000),      # tie at tiny magnitude
        (0x00800000, 0x00800000),      # smallest normal
        (0x00000000, 0x00000000),
        (0x80000000, 0x80000000),      # -0 keeps its sign
        (0x7F800000, 0x7F800000),      # +inf
        (0xFF800000, 0xFF800000),      # -inf
    ]
    x = _f([c[0] for c in cases])
    got = _bits(R.tf32(x))
    want = np.array([c[1] for c in cases], np.uint32)
    assert np.array_equal(got, want), [(hex(a), hex(b), hex(c)) for (a, _), b, c in zip(cases, got, want) if b != c]
    nan = R.tf32(np.array([np.nan], np.float32))
    assert np.isnan(nan).all()


def test_tf32_rounding_properties():
    rs = np.random.RandomState(0)
    x = (rs.standard_normal(100000) * np.exp(rs.uniform(-30, 30, 100000))).astype(np.float32)
    r = R.tf32(x)
    assert (_bits(r) & 0x1FFF == 0).all()                        # 10 mantissa bits
    assert np.array_equal(R.tf32(r), r)                          # idempotent
    assert np.array_equal(R.tf32(-x), -r)                        # symmetric (ties away from zero)
    rel = np.abs(r.astype(np.float64) - x) / np.abs(x.astype(np.float64))
    assert rel.max() <= 2.0 ** -11 * (1 + 1e-6)                  # half an ulp of a 10-bit mantissa
    # nearest: no other 10-bit neighbour is closer
    lo = _f(_bits(x) & np.uint32(0xFFFFE000)).astype(np.float64)
    hi = _f((_bits(x) & np.uint32(0xFFFFE000)) + np.uint32(0x2000)).astype(np.float64)
    d = np.abs(r.astype(np.float64) - x)
    assert (d <= np.minimum(np.abs(lo - x), np.abs(hi - x))).all()
