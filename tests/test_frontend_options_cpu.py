"""Front-end options beyond the shipped configurations, on the CPU: the options oracle against the reference's own outputs
(tests/golden/frontend_options.npz, written by tests/golden/make_frontend_options_golden.py) and against torchaudio,
the featurizer's host constants and frame counts, and the options that keep raising."""
import ctypes
import importlib.util
import os
import warnings

import numpy as np
import pytest
import torch

import frontend_options_oracle as opt
from test_host_logic import _header_struct_fields

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('make_frontend_options_golden',
                                               os.path.join(HERE, 'golden', 'make_frontend_options_golden.py'))
cases = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(cases)


def _fz(method, args):
    from mvector.data_utils.featurizer import AudioFeaturizer
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return AudioFeaturizer(method, method_args=args)


def _oracle(x, ratio, method, args, **kw):
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        return opt.featurize(x, ratio, method, args, **kw)


def test_golden_is_small():
    assert os.path.getsize(os.path.join(HERE, 'golden', 'frontend_options.npz')) < 256 << 10


@pytest.mark.parametrize('i', range(len(cases.CASES)))
def test_oracle_against_reference_golden(i):
    """Tolerances of test_oracle_vs_reference.py: fp32 reductions change order with the CPU's thread count."""
    method, args = cases.CASES[i]
    z = np.load(os.path.join(HERE, 'golden', 'frontend_options.npz'))
    x, ratio, one = cases.front_input()
    fz = _fz(method, args)
    for tag, y in (('batch', _oracle(x, ratio, method, args)), ('single', _oracle(one, None, method, args))):
        y = y.numpy()
        assert list(y.shape) == z[f'case{i}/{tag}/shape'].tolist(), (method, args, tag)
        assert y.shape[1] == fz.num_frames(x.shape[1] if tag == 'batch' else one.numel())
        ref = z[f'case{i}/{tag}/sample']
        d = float(np.abs(y.reshape(-1)[cases.sample_index(y.size, 2 * i + (tag == 'single'))] - ref).max())
        assert d <= 2e-6 * float(np.abs(ref).max()), (method, args, tag, d)
        s, s_ref = y.astype(np.float64).sum(), float(z[f'case{i}/{tag}/sum'])
        assert abs(s - s_ref) <= 1e-6 * float(np.abs(y).astype(np.float64).sum()), (method, args, tag, s, s_ref)
    assert fz.feature_dim == int(z[f'case{i}/feature_dim']) == y.shape[2]


def _torchaudio_features(ta, method, args, w):
    """The reference's transform (before AudioFeaturizer.forward's CMN) straight from torchaudio: [F, T]."""
    if method == 'Fbank':
        return ta.compliance.kaldi.fbank(w[None], **args).T
    return {'MelSpectrogram': ta.transforms.MelSpectrogram, 'Spectrogram': ta.transforms.Spectrogram,
            'MFCC': ta.transforms.MFCC}[method](**args)(w[None])[0]


@pytest.mark.parametrize('i', range(len(cases.CASES)))
def test_oracle_against_torchaudio_at_more_lengths(i):
    ta = pytest.importorskip('torchaudio')
    method, args = cases.CASES[i]
    g = torch.Generator().manual_seed(100 + i)
    for n in (1024, 3201, 7999, 8000, 24011):
        w = torch.randn(n, generator=g) * 0.1
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            ref = _torchaudio_features(ta, method, args, w)
            ours = _oracle(w, None, method, args)[0].T + ref.mean(1, keepdim=True)      # undo the CMN
        assert ours.shape == ref.shape and ours.shape[1] == _fz(method, args).num_frames(n), (method, args, n)
        assert float((ours - ref).abs().max()) <= 2e-6 * float(ref.abs().max()) + 1e-6, (method, args, n)


def test_slaney_and_vtln_banks_and_window_fn_match_torchaudio():
    ta = pytest.importorskip('torchaudio')
    from mvector.data_utils import featurizer as F
    for n_freqs, f_min, f_max, n_mels, sr in ((257, 0.0, 8000.0, 64, 16000), (513, 50.0, 7600.0, 200, 16000),
                                               (201, 20.0, 4000.0, 40, 8000)):
        for norm in (None, 'slaney'):
            for scale in ('htk', 'slaney'):
                with warnings.catch_warnings():
                    warnings.simplefilter('ignore')
                    want = ta.functional.melscale_fbanks(n_freqs, f_min, f_max, n_mels, sr, norm, scale)
                assert torch.equal(F.melscale_fbanks(n_freqs, f_min, f_max, n_mels, sr, norm, scale), want)
    for n_mels, n_fft, sf, lo, hi, vlo, vhi, warp in ((80, 512, 16000.0, 20.0, 0.0, 100.0, -500.0, 0.9),
                                                      (80, 400, 16000.0, 20.0, 0.0, 100.0, -500.0, 1.1),
                                                      (40, 200, 8000.0, 20.0, 3800.0, 300.0, 3000.0, 0.85),
                                                      (23, 512, 16000.0, 20.0, 0.0, 100.0, -500.0, 1.0)):
        want, _ = ta.compliance.kaldi.get_mel_banks(n_mels, n_fft, sf, lo, hi, vlo, vhi, warp)
        assert torch.equal(F.kaldi_mel_banks(n_mels, n_fft, sf, lo, hi, vlo, vhi, warp), want)
    ms = F.MelSpectrogram(n_fft=512, win_length=400, hop_length=160, n_mels=64, window_fn=torch.hamming_window,
                          wkwargs=dict(periodic=False))
    spec = ta.transforms.Spectrogram(n_fft=512, win_length=400, window_fn=torch.hamming_window,
                                     wkwargs=dict(periodic=False))
    assert np.array_equal(ms.window[56:456], spec.window.numpy()) and not ms.window[:56].any()
    assert not ms.window[456:].any()
    sp = F.Spectrogram(n_fft=400, normalized=True)
    assert sp.opts.spec_scale == 1.0 / float(torch.hann_window(400).pow(2.0).sum().sqrt())
    assert F.Spectrogram(n_fft=512, normalized='frame_length').opts.spec_scale == 1.0 / np.sqrt(512)


def _boundary_lengths(WL, hop, n_fft, pad):
    half = n_fft // 2
    out = {WL, WL + 1, 2 * WL, hop // 2, hop // 2 + 1, half - 2 * pad, half + 1 - 2 * pad, half + 2 - 2 * pad,
           n_fft - 2 * pad, n_fft + 1 - 2 * pad}
    for k in (3, 10, 31):
        out |= {k * hop - 1, k * hop, k * hop + 1, k * hop + hop // 2 - 1, k * hop + hop // 2}
    return sorted(n for n in out if n >= 1)


@pytest.mark.parametrize('method,args', [
    ('Fbank', dict(num_mel_bins=40)),
    ('Fbank', dict(num_mel_bins=40, snip_edges=False)),
    ('Fbank', dict(num_mel_bins=40, snip_edges=False, round_to_power_of_two=False, frame_shift=12.5)),
    ('Fbank', dict(num_mel_bins=40, snip_edges=False, frame_length=8.0, frame_shift=12.0)),      # pad < 0: trimmed front
    ('Spectrogram', dict(n_fft=400, hop_length=160)),
    ('Spectrogram', dict(n_fft=400, hop_length=160, center=False)),
    ('Spectrogram', dict(n_fft=256, hop_length=100, center=False, pad=30)),
    ('Spectrogram', dict(n_fft=256, hop_length=100, pad=7, pad_mode='circular')),
    ('Spectrogram', dict(n_fft=256, hop_length=100, pad=7, pad_mode='constant')),
    ('Spectrogram', dict(n_fft=256, hop_length=100, pad_mode='replicate')),
])
def test_num_frames_follows_the_framing_at_boundary_lengths(method, args):
    """AudioFeaturizer.num_frames (evaluate's .npy crop, predict's batching) against the oracle's shapes, and lengths
    that break torch's precondition raise in the oracle (so the featurizer's device call must refuse them too)."""
    fz = _fz(method, args)
    f = fz.feat_fun
    pad = f.opts.pad if f.desc.kind == 1 else 0
    for n in _boundary_lengths(f.win_length if f.desc.kind == 0 else f.n_fft, f.hop, f.n_fft, pad):
        w = torch.randn(n, generator=torch.Generator().manual_seed(n)) * 0.1
        try:
            T = _oracle(w, None, method, args).shape[1]
        except (AssertionError, RuntimeError):
            T = None
        if f.desc.kind == 0:
            valid = 2 <= f.win_length <= n
        else:
            Lp, half = n + 2 * pad, f.n_fft // 2
            valid = {0: half < Lp, 4: half <= Lp, 5: f.n_fft <= Lp}.get(f.opts.frame_mode, True)
        assert (T is not None) == valid, (method, args, n)
        if valid:
            assert fz.num_frames(n) == T, (method, args, n)


def test_subtract_mean_is_the_existing_cmn():
    """subtract_mean's per-utterance column mean is subtracted again by AudioFeaturizer.forward: the result is plain CMN
    up to rounding, so the lowering needs no kernel change."""
    w = torch.randn(2, 48000, generator=torch.Generator().manual_seed(3)) * 0.1
    args = dict(sample_frequency=16000, num_mel_bins=80)
    a = _oracle(w, None, 'Fbank', dict(args, subtract_mean=True))
    b = _oracle(w, None, 'Fbank', args)
    assert float((a - b).abs().max()) <= 1e-6 and float(b.abs().max()) > 4.0
    fz = _fz('Fbank', dict(args, subtract_mean=True))
    assert fz.feat_fun.opts.frame_mode == 0 and fz.num_frames(48000) == 298


@pytest.mark.parametrize('method,args,name', [
    ('Fbank', dict(dither=0.1), 'dither'),
    ('Fbank', dict(min_duration=0.5), 'min_duration'),
    ('Fbank', dict(channel=1), 'channel'),
    ('Fbank', dict(use_energy=True), 'use_energy'),
    ('Fbank', dict(round_to_power_of_two=False, frame_length=26.0), 'round_to_power_of_two'),     # 416 = 2^5 13
    ('MelSpectrogram', dict(power=3.0), 'power'),
    ('MelSpectrogram', dict(n_fft=442), 'n_fft'),
    ('MelSpectrogram', dict(n_fft=4096), 'n_fft'),
    ('MelSpectrogram', dict(n_fft=256, n_mels=130), 'n_mels'),
    ('Spectrogram', dict(onesided=False), 'onesided'),
    ('Spectrogram', dict(power=None), 'power'),
    ('MFCC', dict(melkwargs=dict(n_fft=1024, n_mels=160)), 'n_mels'),
])
def test_unsupported_options_raise_naming_the_option(method, args, name):
    with pytest.raises(NotImplementedError, match=name):
        _fz(method, args)


def test_invalid_values_raise_what_the_reference_raises():
    with pytest.raises(ValueError):
        _fz('Spectrogram', dict(normalized='bogus'))
    with pytest.raises(ValueError):
        _fz('MelSpectrogram', dict(norm='bogus'))
    with pytest.raises(ValueError):
        _fz('MelSpectrogram', dict(mel_scale='bogus'))
    with pytest.raises(NotImplementedError, match='padding mode'):
        _fz('MelSpectrogram', dict(pad_mode='bogus'))
    with pytest.raises(AssertionError):
        _fz('Fbank', dict(vtln_warp=0.9, vtln_low=10.0))                 # vtln_low must exceed low_freq
    with pytest.raises(TypeError):
        _fz('Spectrogram', dict(n_mels=40))
    # options that only matter with use_energy are accepted without it, as the reference ignores them
    assert _fz('Fbank', dict(raw_energy=False, energy_floor=0.0, htk_compat=True)).feature_dim == 23


def test_ctypes_options_struct_follows_the_header():
    from mvector import _lib
    ctype_of = {'int32_t': ctypes.c_int32, 'double': ctypes.c_double}
    want = _header_struct_fields('vp_frontend_options')
    got = list(_lib.FrontendOptions._fields_)
    assert [(n, ctype_of[t]) for t, n, _ in want] == got
    assert ctypes.sizeof(_lib.FrontendOptions) == 16
