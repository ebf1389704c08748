"""Op-level GPU tests of the fused front-end (frontend_kernel, mfcc_post_kernel, max_reduce_kernel, cmn_mask_kernel) at
the plan branches where it goes wrong: every instantiation on both kinds, 1 / 2 / 4 tiles per CTA with and without the
on-chip feature cache, the plain and 4-chain mel projections, both frame-mean paths, every framing mode across the
ends of a CTA's span, the CMN mask at its edges and the MFCC reductions past their first sweep.

Each case of tests/frontend_cases.py first asserts the plan it runs (vp_frontend_plan_info == the host-plan mirror ==
the case's intent), then compares one call with the fp64 reference ``exact_features``.  Bars: Fbank absolute in log
units; MelSpectrogram / Spectrogram relative to the frame scale (its maximum, or the CMN mean it is shifted by when
that is larger); MFCC relative to max|ref|.  Masked frames are +0.0 bits and a second call is bit-identical.

The errors quoted were measured on an H100 80GB HBM3 (700 W); the module runs in about 15 s there."""
import ctypes as C

import numpy as np
import pytest
import torch

import frontend_cases as fc
from mvector import _lib as L

pytestmark = pytest.mark.gpu

# Measured maxima over the cases (H100 80GB HBM3): Fbank 9.7e-6 (log units), MelSpectrogram 1.5e-7, Spectrogram 6.6e-8
# (relative to the frame scale), MFCC 1.2e-6 (relative to max|ref|, on mfcc_many_ctas_loud_last; <= 6.2e-7 on the rest).
# The results are bit-deterministic.  With the twiddle table and the radix-5 / 3 roots rounded to fp32 the Fbank cases
# reach 2.8e-5 and both Spectrogram cases 1.3e-7 / 1.4e-7, so those two bars fail; MelSpectrogram moves to 2.3e-7 at
# most while its clean maximum is 1.5e-7 (the same case measures 1.5e-7 both ways), so no MelSpectrogram bar
# separates the two.
BARS = dict(Fbank=1.2e-5, MelSpectrogram=1e-6, Spectrogram=1e-7, MFCC=3e-6)


@pytest.fixture(scope='module')
def engine():
    from mvector.engine import Engine
    eng = Engine()
    yield eng
    eng.close()


def _featurizer(name, engine):
    from mvector.data_utils.featurizer import AudioFeaturizer
    c = fc.CASES[name]
    fz = AudioFeaturizer(c['method'], method_args=c['args'], engine=engine)
    fz.engine                                         # configure the handle (vp_frontend_set + options)
    return fz


def _plan_info(fz, B, Lpad):
    info = (C.c_int32 * 8)()
    stage = fz.feat_fun.desc.post
    assert L.lib().vp_frontend_plan_info(fz.engine.handle, B, Lpad, stage, info) == L.VP_OK
    got = dict(zip(fc.PLAN_KEYS, list(info)))
    got['mel'] = ('plain', 'chain4')[got['mel']]
    return got


def _err(method, got, ref, scale):
    d = np.abs(got.astype(np.float64) - ref)
    if method == 'Fbank':
        return float(d.max())
    if method == 'MFCC':
        return float(d.max() / np.abs(ref).max())
    return float((d / np.maximum(scale, 1e-30)[..., None]).max())


@pytest.mark.parametrize('name', list(fc.CASES))
def test_frontend_case(name, engine):
    """One call per case against the fp64 reference, its plan asserted first.  Measured maxima (H100 80GB HBM3):
    Fbank 9.7e-6 (fbank80_512_tpc1_residues), MelSpectrogram 1.5e-7, Spectrogram 6.6e-8, MFCC 1.2e-6
    (mfcc_many_ctas_loud_last)."""
    c = fc.CASES[name]
    x, ratio, keep, T = fc.materialize(name)
    B, Lpad = x.shape
    fz = _featurizer(name, engine)
    plan = fc.plan_of(name)
    assert _plan_info(fz, B, Lpad) == {k: plan[k] for k in fc.PLAN_KEYS}
    assert {k: plan[k] for k in c['intent']} == c['intent']
    xd = torch.from_numpy(x).cuda()
    got = fz(xd, ratio).cpu().numpy()
    again = fz(xd, ratio).cpu().numpy()
    assert got.shape == (B, T, fz.feature_dim)
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32))
    ref, scale = fc.exact_features(c['method'], c['args'], x, keep)
    err = _err(c['method'], got, ref, scale)
    print(f'{name}: {c["method"]} err {err:.3e}')
    assert err <= BARS[c['method']], (name, err)
    if keep is not None:
        for b, k in enumerate(keep):
            assert not got[b, k:].view(np.uint32).any()       # +0.0 bits


def test_mfcc_two_stage_matches_one_stage(engine):
    """vp_mfcc_mel + vp_mfcc_finish (the sharded MFCC's two halves, here on one process) are bit-identical to
    vp_features on the case with 320 per-CTA maxima whose largest sits at index >= 304: max_reduce_kernel must read past
    its first 256."""
    name = fc.TWO_STAGE
    c = fc.CASES[name]
    x, _, _, T = fc.materialize(name)
    B, Lpad = x.shape
    fz = _featurizer(name, engine)
    lib, h = L.lib(), fz.engine.handle
    xd = torch.from_numpy(x).cuda()
    one = fz(xd).cpu().numpy()
    scratch = torch.empty(int(lib.vp_frontend_scratch_floats(h, B, Lpad)), device='cuda')
    feats = torch.full((B, T, fz.feature_dim), float('nan'), device='cuda')
    mx = torch.empty(1, device='cuda')
    st = fz.engine.stream_ptr()
    assert lib.vp_mfcc_mel(h, C.c_void_p(xd.data_ptr()), B, Lpad, C.c_void_p(scratch.data_ptr()),
                           C.c_void_p(mx.data_ptr()), st) == L.VP_OK
    assert lib.vp_mfcc_finish(h, B, Lpad, C.c_void_p(), C.c_void_p(feats.data_ptr()), C.c_void_p(scratch.data_ptr()),
                              C.c_void_p(mx.data_ptr()), st) == L.VP_OK
    two = feats.cpu().numpy()
    assert np.array_equal(one.view(np.uint32), two.view(np.uint32))
    ref, scale = fc.exact_features(c['method'], c['args'], x)
    assert _err('MFCC', two, ref, scale) <= BARS['MFCC']
