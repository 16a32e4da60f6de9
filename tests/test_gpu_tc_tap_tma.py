"""The strided stage convolutions' taps by TMA in the tensor-core GEMM core (csrc/gemm_tc.cuh, tc_seg_tma and
tc_encode_taps): on the strided schedule a stage's frame map is affine across clips, so each stage of the conv's taps
and of the 1x1 layer's A arrives as one 4D TMA box {32, J, 1, fpt} instead of a per-row cp.async gather.

- every GEMM launch of a strided model's forward, audited by tests/gemmaudit.py (each launch against fp64 of its own
  operands, the output columns it does not own unchanged), at J = 15, 16, 17, 19 (8, 8, 7 and 6 frames per tile),
  stage widths Cw = 32, 64, 128, 256, 3 and 5 taps, stage-1 tile counts below, at and well above the SM count with a
  partial last row tile, in F16X3 and 1xTF32 (inference) and 3xTF32 (the training forward); the stage conv and the
  1x1 + residual launches are asserted to be fed by TMA;
- schedule independence: the headline model's first 8 clips are bitwise the same in a forward of 4096 clips and in
  one of those 8 alone."""
import numpy as np
import pytest
import torch

from gast_b200 import _lib, engine, synth
import gemmaudit as GA

pytestmark = pytest.mark.gpu

# (J, filter widths, channels): stage widths Cw = channels << i; stage 1 runs 3 taps at J = 15 and 17 and 5 at J = 16
# and 19 (the model takes odd widths only), stage 2 3 taps
GEOMETRIES = [(15, [3, 3, 3], 16), (16, [3, 5, 3], 64), (17, [3, 3, 3], 64), (19, [3, 5, 3], 16)]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _clips(J, fw, ch, where):
    """clips whose stage-1 GEMMs run below, at or well above one tile per SM, with a partial last row tile"""
    fpt = 128 // J
    col_tiles = ((ch << 1) + 127) // 128
    t1 = int(np.prod(fw[2:]))                               # stage-1 output frames per clip
    sms = _sms()
    want = {'below': sms // 3, 'at': sms, 'above': 2 * sms + 9}[where]
    for B in range(1, 20000):
        F = B * t1
        if F % fpt and ((F + fpt - 1) // fpt) * col_tiles >= want:
            return B
    raise AssertionError('no clip count reaches %d tiles' % want)


def _model(J, fw, ch):
    from model.gast_net import SpatioTemporalModelOptimized1f
    import fp64ref as R
    m = SpatioTemporalModelOptimized1f(R.adj(J), J, 2, J, fw, dropout=0.0, channels=ch)
    synth.randomize_module(m, J + ch)
    return m.cuda()


def _audited(m, fn):
    fn()                                                     # creates the handle
    h = list(m.__dict__['_gast_handles'].values())[0]
    aud = GA.Auditor()
    aud.install(h.lib, h.h)
    try:
        try:
            fn()
        except engine.GastError as ex:
            raise AssertionError('%s\n%s' % (ex, aud.failure)) from ex
        torch.cuda.synchronize()
    finally:
        h.lib.gast_debug_set_gemm_audit(h.h, _lib.GemmAuditFn(), None)
    assert aud.failure is None, aud.failure
    assert aud.records
    return aud.records


def _check_stage_feed(recs, fw, ch, form, res=True):
    """the stage convolutions (and, in inference, the 1x1 + residual launches) ran on the tensor cores, fed by TMA"""
    conv = [r for r in recs if r['core'] == 'tc' and 'tap_stride_t_mul' in r['shape']]
    assert len(conv) == len(fw) - 1, [r['shape'] for r in conv]
    for i, c in enumerate(conv):
        Cw = ch << (i + 1)
        assert c['form'] == form and c['N'] == Cw and c['K'] == fw[i + 1] * Cw and c['tma_mask'] == 1, c
    assert 'partial_row_tile' in conv[0]['shape']
    if res:
        r1 = [r for r in recs if 'res_map' in r['shape']]
        assert len(r1) == len(fw) - 1 and all(r['core'] == 'tc' and r['tma_mask'] == 1 for r in r1), r1


@pytest.mark.parametrize('prec,where', [('fp32', 'below'), ('fp32', 'at'), ('fp32', 'above'), ('tf32', 'below'),
                                        ('tf32', 'above')])
@pytest.mark.parametrize('geo', range(len(GEOMETRIES)))
def test_inference_stages(prec, geo, where):
    J, fw, ch = GEOMETRIES[geo]
    B = _clips(J, fw, ch, where)
    T = int(np.prod(fw))
    m = engine.set_precision(_model(J, fw, ch).eval(), prec)
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=B)).cuda()

    def fwd():
        with torch.no_grad():
            return m(x).clone()
    recs = _audited(m, fwd)
    _check_stage_feed(recs, fw, ch, 'f16x3' if prec == 'fp32' else 'tf32')


@pytest.mark.parametrize('where', ['below', 'above'])
@pytest.mark.parametrize('geo', range(len(GEOMETRIES)))
def test_training_forward_stages(geo, where):
    J, fw, ch = GEOMETRIES[geo]
    B = _clips(J, fw, ch, where)
    T = int(np.prod(fw))
    m = engine.set_training_precision(_model(J, fw, ch).train(), 'fp32')
    x = torch.from_numpy(synth.synth_input(B, T, J, 2, seed=B)).cuda()

    def fwd():
        return m(x).detach().clone()
    recs = _audited(m, fwd)
    _check_stage_feed(recs, fw, ch, '3xtf32', res=False)     # training adds the residual in its BatchNorm pass


def test_headline_schedule_independent():
    from test_gpu_forward_fp64 import HEADLINE, HEADLINE_B, build_model
    m = build_model(*HEADLINE, seed=1).cuda()
    x = torch.from_numpy(synth.synth_input(HEADLINE_B, 27, 17, 2, seed=1234)).cuda()
    with torch.no_grad():
        y_all = m(x)[:8].cpu().numpy()
        y_8 = m(x[:8].contiguous()).cpu().numpy()
    assert np.array_equal(y_all.view(np.uint32), y_8.view(np.uint32))
