"""Front-end options beyond the shipped configurations on the device (run on an H100: python -m pytest tests -m gpu):
every option case of tests/golden/make_frontend_options_golden.py through AudioFeaturizer against the options oracle,
the default framing spelled out explicitly, the options' reset and two-stage MFCC, length preconditions, and two
end-to-end embeddings through MVectorPredictor.predict_batch."""
import ctypes as C
import importlib.util
import os
import tempfile
import warnings

import numpy as np
import pytest
import torch

import frontend_options_oracle as opt
from conftest import load_golden, rel_l2
from test_gpu_parity import EMB_TOL, FBANK_ABS_TOL, FBANK_EXACT_TOL, _cfg

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_frontend_options_golden',
                                               os.path.join(HERE, 'golden', 'make_frontend_options_golden.py'))
cases = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(cases)


def _fz(method, args):
    from mvector.data_utils.featurizer import AudioFeaturizer
    return AudioFeaturizer(method, method_args=args)


def _oracle(x, ratio, method, args, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return opt.featurize(x, ratio, method, args, **kw)


def _check(got, x, ratio, method, args):
    ref = _oracle(x, ratio, method, args)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if method == 'Fbank':           # the three-way bar of test_gpu_parity.py
        exact = _oracle(x, ratio, method, args, exact_spectrum=True)
        e_got, e_ref, d = [float((a - b).abs().max()) for a, b in ((got, exact), (ref, exact), (got, ref))]
        assert e_got <= FBANK_EXACT_TOL and d <= e_ref + FBANK_EXACT_TOL and d < FBANK_ABS_TOL, (e_got, d, e_ref)
    else:
        tol = 2e-5 if method == 'MFCC' else 3e-6          # relative to the range (one frame: CMN leaves zeros)
        assert float((got - ref).abs().max()) <= tol * float(ref.abs().max())
    return ref


@pytest.mark.parametrize('i', range(len(cases.CASES)))
def test_option_case_on_device(i):
    from mvector import _lib as L
    method, args = cases.CASES[i]
    x, ratio, one = cases.front_input()
    fz = _fz(method, args)
    got = fz(x, ratio).cpu()
    ref = _check(got, x, ratio, method, args)
    keep = torch.round(ratio * ref.shape[1]).long()
    for b, k in enumerate(keep.tolist()):
        assert torch.all(got[b, k:] == 0)                      # masked frames are exactly zero
    got1 = fz(one).cpu()
    _check(got1, one, None, method, args)
    h = fz.engine.handle
    for n, T in ((x.shape[1], got.shape[1]), (one.numel(), got1.shape[1])):
        assert L.lib().vp_num_frames(h, n) == fz.num_frames(n) == T


SHIPPED = [
    ('Fbank', dict(sample_frequency=16000, num_mel_bins=80),
     dict(snip_edges=True, round_to_power_of_two=True, subtract_mean=False, vtln_warp=1.0, dither=0.0)),
    ('MelSpectrogram', dict(sample_rate=16000, n_fft=1024, win_length=1024, hop_length=320, f_min=50.0, f_max=14000.0,
                            n_mels=64),
     dict(center=True, pad_mode='reflect', pad=0, normalized=False, norm=None, mel_scale='htk',
          window_fn=torch.hann_window)),
    ('Spectrogram', dict(), dict(center=True, pad_mode='reflect', pad=0, normalized=False, onesided=True)),
    ('MFCC', dict(), dict(melkwargs=dict(center=True, pad_mode='reflect', normalized=False, mel_scale='htk'))),
]


@pytest.mark.parametrize('method,args,explicit', SHIPPED, ids=[s[0] for s in SHIPPED])
def test_explicit_defaults_are_bit_identical(method, args, explicit):
    x, ratio, _ = cases.front_input()
    a = _fz(method, args)(x, ratio).cpu()
    b = _fz(method, dict(args, **explicit))(x, ratio).cpu()
    assert torch.equal(a, b)


def test_frontend_set_restores_the_default_framing():
    from mvector import _lib as L
    from mvector.engine import _check as check
    args = dict(n_fft=512, hop_length=160, n_mels=64)
    x, ratio, _ = cases.front_input()
    fz = _fz('MelSpectrogram', dict(args, center=False, normalized=True))
    fz(x, ratio)
    f, lib, h = fz.feat_fun, L.lib(), fz.engine.handle
    start, count, off, w = f.bank
    check(h, lib.vp_frontend_set(h, C.byref(f.desc), f.window.ctypes.data_as(C.c_void_p),
                                 start.ctypes.data_as(C.c_void_p), count.ctypes.data_as(C.c_void_p),
                                 off.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p), int(w.size), None))
    B, Lp = x.shape
    T = 1 + Lp // 160
    assert lib.vp_num_frames(h, Lp) == T
    wd = x.cuda().contiguous()
    feats = torch.empty(B, T, 64, device='cuda')
    scratch = torch.empty(int(lib.vp_frontend_scratch_floats(h, B, Lp)), device='cuda')
    check(h, lib.vp_melspec(h, C.c_void_p(wd.data_ptr()), B, Lp, None, C.c_void_p(feats.data_ptr()),
                            C.c_void_p(scratch.data_ptr()), fz.engine.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(feats.cpu(), _fz('MelSpectrogram', args)(x).cpu())


def test_two_stage_mfcc_honours_the_options():
    args = dict(n_mfcc=24, melkwargs=dict(n_fft=512, hop_length=160, n_mels=64, center=False, pad=30,
                                          normalized='frame_length'))
    x, ratio, _ = cases.front_input()
    fz = _fz('MFCC', args)
    one_call = fz(x, ratio)
    w = x.cuda().contiguous()
    B, Lp = w.shape
    keep = fz.keep_frames(ratio, fz.num_frames(Lp)).cuda()
    from mvector import _lib as L
    feats = torch.empty_like(one_call)
    scratch = torch.empty(int(L.lib().vp_frontend_scratch_floats(fz.engine.handle, B, Lp)), device='cuda')
    fz.mfcc_sharded(w, B, Lp, C.c_void_p(keep.data_ptr()), feats, scratch, torch.cuda.current_stream(), None)
    torch.cuda.synchronize()
    assert torch.equal(feats, one_call)


def test_lengths_that_break_a_precondition_raise_before_any_launch():
    from mvector._lib import VpError
    cases_ = [('Spectrogram', dict(n_fft=400, center=False), 399, 400),
              ('Spectrogram', dict(n_fft=400), 200, 201),                                 # reflect: n_fft/2 < L
              ('Spectrogram', dict(n_fft=400, pad_mode='circular'), 199, 200),            # circular: n_fft/2 <= L
              ('MelSpectrogram', dict(n_fft=512, n_mels=40, center=False, pad=6), 499, 500)]
    for method, args, bad, good in cases_:
        fz = _fz(method, args)
        with pytest.raises(VpError):
            fz(torch.randn(1, bad))
        w = torch.randn(1, good)
        _check(fz(w).cpu(), w, None, method, args)
    with pytest.raises(AssertionError):                                                   # kaldi.py: window <= L
        _fz('Fbank', dict(num_mel_bins=40, snip_edges=False))(torch.randn(1, 399))


@pytest.mark.parametrize('prep', [
    dict(feature_method='Fbank', method_args=dict(sample_frequency=16000, num_mel_bins=80, snip_edges=False,
                                                  round_to_power_of_two=False)),
    dict(feature_method='MelSpectrogram', method_args=dict(sample_rate=16000, n_fft=512, win_length=400, hop_length=160,
                                                           n_mels=80, center=False, norm='slaney', mel_scale='slaney',
                                                           normalized=True)),
], ids=['fbank', 'melspectrogram'])
def test_predict_batch_end_to_end(prep, manifest):
    """Waveforms -> embeddings through the drop-in predictor on the small golden ECAPA weights (80-wide input), against
    the options oracle's features through the CPU oracle model."""
    from mvector.predict import MVectorPredictor
    from oracle import frontend as ofe, models as om
    m = manifest['ecapa_small']
    z, sd = load_golden('ecapa_small')
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        pred = MVectorPredictor(configs=_cfg(m['model'], m['model_args'], prep), model_path=td, use_gpu=True)
    waves = [z['wave%d' % i] for i in range(len(m['lens']))]
    emb = pred.predict_batch(waves)
    x, ratio = ofe.pad_batch(waves)
    feats = _oracle(x, ratio, prep['feature_method'], prep['method_args'])
    ref = om.forward(m['model'], sd, feats, **m['model_args']).numpy()
    assert rel_l2(emb, ref).max() < EMB_TOL
