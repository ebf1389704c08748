"""AudioFeaturizer mirror (reference: mvector/data_utils/featurizer.py:9-132), backed by the fused sm_90a front-end.

Host side only prepares constants once (window, sparse mel bank, DCT matrix -- the reference rebuilds the Kaldi ones on
every call, kaldi.py:201,621-627) and hands device pointers to ``vp_features`` (``AudioFeaturizer.launch``); the
per-utterance Python loop (featurizer.py:124-131), the transpose, the CMN and the length mask (featurizer.py:77-90) all
run in two kernels (three for MFCC).  All four ``feature_method`` values of the reference are lowered: Fbank,
MelSpectrogram, Spectrogram (pass-through bank over the n_fft/2+1 bins) and MFCC.
"""
import ctypes as C
import math

import numpy as np
import torch
from loguru import logger

from .. import _lib as L
from ..engine import Engine, _check

_FBANK_DEFAULTS = dict(blackman_coeff=0.42, channel=-1, dither=0.0, energy_floor=1.0, frame_length=25.0,
                       frame_shift=10.0, high_freq=0.0, htk_compat=False, low_freq=20.0, min_duration=0.0,
                       num_mel_bins=23, preemphasis_coefficient=0.97, raw_energy=True, remove_dc_offset=True,
                       round_to_power_of_two=True, sample_frequency=16000.0, snip_edges=True, subtract_mean=False,
                       use_energy=False, use_log_fbank=True, use_power=True, vtln_high=-500.0, vtln_low=100.0,
                       vtln_warp=1.0, window_type='povey')
_MELSPEC_DEFAULTS = dict(sample_rate=16000, n_fft=400, win_length=None, hop_length=None, f_min=0.0, f_max=None,
                         pad=0, n_mels=128, power=2.0, normalized=False, center=True, pad_mode='reflect',
                         onesided=None, norm=None, mel_scale='htk')
_SPEC_DEFAULTS = dict(n_fft=400, win_length=None, hop_length=None, pad=0, power=2.0, normalized=False, center=True,
                      pad_mode='reflect', onesided=True)
_MFCC_DEFAULTS = dict(sample_rate=16000, n_mfcc=40, dct_type=2, norm='ortho', log_mels=False, melkwargs=None)


def _fft_size_ok(n):
    """The front-end FFT handles N = 2^a 3^b 5^c, 4 | N, 64 <= N <= 2048 (torchaudio's default n_fft = 400 included)."""
    if n < 64 or n > 2048 or n % 4:
        return False
    for f in (2, 3, 5):
        while n % f == 0:
            n //= f
    return n == 1


def _sparse_bank(dense):
    """dense [n_filters, n_bins] -> (start, count, offset, weights) over each filter's non-zero support."""
    start, count, off, w = [], [], [], []
    for row in dense:
        nz = np.nonzero(row)[0]
        if nz.size == 0:
            start.append(0); count.append(0); off.append(len(w))
            continue
        s, e = int(nz[0]), int(nz[-1]) + 1
        start.append(s); count.append(e - s); off.append(len(w))
        w.extend(row[s:e].tolist())
    return (np.asarray(start, np.int32), np.asarray(count, np.int32), np.asarray(off, np.int32),
            np.asarray(w if w else [0.0], np.float32))


def _unsupported(method, bad):
    """Options outside the lowered front-end raise, each named with the reason: there is no CPU fallback."""
    if bad:
        raise NotImplementedError(f'{method} options not lowered to the sm_90a front-end: ' + '; '.join(bad))


_FFT_SIZES = 'the FFT handles 2^a 3^b 5^c, a multiple of 4, in [64, 2048]'


def _stft_window(n_fft, win_length, window_fn=torch.hann_window, wkwargs=None):
    """window_fn(win_length, **wkwargs) (torchaudio's Spectrogram; periodic Hann by default), centred inside n_fft like
    torch.stft does for a short window.  -> (the n_fft taps, the win_length taps before the padding)."""
    taps = (window_fn(win_length) if wkwargs is None else window_fn(win_length, **wkwargs)).to(torch.float32)
    win = taps
    if win_length < n_fft:
        left = (n_fft - win_length) // 2
        win = torch.nn.functional.pad(win, (left, n_fft - win_length - left))
    return win.numpy().astype(np.float32), taps


_PAD_MODES = {'reflect': L.FRAME_DEFAULT, 'constant': L.FRAME_STFT_CONSTANT, 'replicate': L.FRAME_STFT_REPLICATE,
              'circular': L.FRAME_STFT_CIRCULAR}


def _stft_options(a, n_fft, taps):
    """Framing and scale of torchaudio's spectrogram (functional.py:52-144): zeros `pad` (> 0 only) at both ends, then
    torch.stft centring by n_fft/2 in `pad_mode` (none when center=False), and |X| scaled by 1/sqrt(sum(window^2))
    (normalized True / 'window') or by 1/sqrt(n_fft) (normalized 'frame_length', torch.stft's own normalisation)."""
    normalized = a['normalized']
    if isinstance(normalized, str):
        if normalized not in ('frame_length', 'window'):
            raise ValueError('Invalid normalized parameter: {}'.format(normalized))
    elif not isinstance(normalized, bool):
        raise TypeError('Input type not supported')
    if normalized == 'frame_length':
        scale = 1.0 / math.sqrt(n_fft)
    elif normalized is True or normalized == 'window':
        scale = 1.0 / float(taps.pow(2.0).sum().sqrt())      # the fp32 norm the reference divides by
    else:
        scale = 1.0
    if not a['center']:
        mode = L.FRAME_STFT_NOCENTER
    elif a['pad_mode'] in _PAD_MODES:
        mode = _PAD_MODES[a['pad_mode']]
    else:
        raise NotImplementedError('Unrecognised padding mode ' + str(a['pad_mode']))
    return L.FrontendOptions(frame_mode=mode, pad=max(int(a['pad']), 0), spec_scale=scale)


def _hz_to_mel(f, mel_scale):
    """functional._hz_to_mel (functional.py:425-456), python floats."""
    if mel_scale == 'htk':
        return 2595.0 * math.log10(1.0 + (f / 700.0))
    mels = f / (200.0 / 3)
    if f >= 1000.0:
        mels = 1000.0 / (200.0 / 3) + math.log(f / 1000.0) / (math.log(6.4) / 27.0)
    return mels


def _mel_to_hz(mels, mel_scale):
    """functional._mel_to_hz (functional.py:459-489), fp32 tensor."""
    if mel_scale == 'htk':
        return 700.0 * (10.0 ** (mels / 2595.0) - 1.0)
    min_log_mel, logstep = 1000.0 / (200.0 / 3), math.log(6.4) / 27.0
    freqs = 0.0 + (200.0 / 3) * mels
    log_t = mels >= min_log_mel
    freqs[log_t] = 1000.0 * torch.exp(logstep * (mels[log_t] - min_log_mel))
    return freqs


def melscale_fbanks(n_freqs, f_min, f_max, n_mels, sample_rate, norm=None, mel_scale='htk'):
    """functional.melscale_fbanks (functional.py:518-587): HTK or Slaney mel scale, optional Slaney area normalisation.
    Returns [n_freqs, n_mels] float32."""
    if norm is not None and norm != 'slaney':
        raise ValueError('norm must be one of None or "slaney"')
    if mel_scale not in ('htk', 'slaney'):
        raise ValueError('mel_scale should be one of "htk" or "slaney".')
    all_freqs = torch.linspace(0, sample_rate // 2, n_freqs)
    f_pts = _mel_to_hz(torch.linspace(_hz_to_mel(f_min, mel_scale), _hz_to_mel(f_max, mel_scale), n_mels + 2),
                       mel_scale)
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts.unsqueeze(0) - all_freqs.unsqueeze(1)
    fb = torch.max(torch.zeros(1), torch.min((-1.0 * slopes[:, :-2]) / f_diff[:-1], slopes[:, 2:] / f_diff[1:]))
    if norm == 'slaney':
        fb *= (2.0 / (f_pts[2:n_mels + 2] - f_pts[:n_mels])).unsqueeze(0)
    return fb


def _kaldi_mel(f):
    return 1127.0 * (1.0 + f / 700.0).log()


def _vtln_warp_freq(vtln_low, vtln_high, low_freq, high_freq, warp, freq):
    """kaldi.vtln_warp_freq (kaldi.py:334-406): identity outside [low_freq, high_freq], freq / warp between the
    inflection points l = vtln_low * max(1, warp) and h = vtln_high * min(1, warp), linear in between."""
    assert vtln_low > low_freq, 'be sure to set the vtln_low option higher than low_freq'
    assert vtln_high < high_freq, 'be sure to set the vtln_high option lower than high_freq [or negative]'
    lo, hi = vtln_low * max(1.0, warp), vtln_high * min(1.0, warp)
    scale = 1.0 / warp
    assert lo > low_freq and hi < high_freq
    scale_left = (scale * lo - low_freq) / (lo - low_freq)
    scale_right = (high_freq - scale * hi) / (high_freq - hi)
    res = torch.empty_like(freq)
    outside = torch.lt(freq, low_freq) | torch.gt(freq, high_freq)
    before_l, before_h, after_h = torch.lt(freq, lo), torch.lt(freq, hi), torch.ge(freq, hi)
    res[after_h] = high_freq + scale_right * (freq[after_h] - high_freq)       # later masks overwrite earlier ones
    res[before_h] = scale * freq[before_h]
    res[before_l] = low_freq + scale_left * (freq[before_l] - low_freq)
    res[outside] = freq[outside]
    return res


def kaldi_mel_banks(n_mels, n_fft, sf, low_freq, high_freq, vtln_low=100.0, vtln_high=-500.0, vtln_warp=1.0):
    """kaldi.get_mel_banks (kaldi.py:436-511), VTLN-warped when vtln_warp != 1.  Returns [n_mels, n_fft // 2] float32."""
    nyq = 0.5 * sf
    if high_freq <= 0.0:
        high_freq += nyq
    assert 0.0 <= low_freq < nyq and 0.0 < high_freq <= nyq and low_freq < high_freq, \
        'Bad values in options: low-freq / high-freq'
    bw = sf / n_fft
    mlo, mhi = 1127.0 * math.log(1.0 + low_freq / 700.0), 1127.0 * math.log(1.0 + high_freq / 700.0)
    delta = (mhi - mlo) / (n_mels + 1)
    if vtln_high < 0.0:
        vtln_high += nyq
    assert vtln_warp == 1.0 or (low_freq < vtln_low < high_freq and 0.0 < vtln_high < high_freq
                                and vtln_low < vtln_high), 'Bad values in options: vtln-low / vtln-high'
    b = torch.arange(n_mels).unsqueeze(1)
    left, center, right = mlo + b * delta, mlo + (b + 1.0) * delta, mlo + (b + 2.0) * delta
    if vtln_warp != 1.0:
        left, center, right = (_kaldi_mel(_vtln_warp_freq(vtln_low, vtln_high, low_freq, high_freq, vtln_warp,
                                                          700.0 * ((x / 1127.0).exp() - 1.0)))
                               for x in (left, center, right))
    mel = _kaldi_mel(bw * torch.arange(n_fft / 2)).unsqueeze(0)
    up, down = (mel - left) / (center - left), (right - mel) / (right - center)
    if vtln_warp == 1.0:
        return torch.max(torch.zeros(1), torch.min(up, down))
    banks = torch.zeros_like(up)                          # warping can reorder left / center / right
    up_idx = torch.gt(mel, left) & torch.le(mel, center)
    down_idx = torch.gt(mel, center) & torch.lt(mel, right)
    banks[up_idx] = up[up_idx]
    banks[down_idx] = down[down_idx]
    return banks


class KaldiFbank:
    """kwargs of torchaudio.compliance.kaldi.fbank (featurizer.py:114-117); constants follow kaldi.py:86-113
    (window) and kaldi.py:436-511 (mel banks, VTLN-warped or not), evaluated once in fp32 with the same torch ops.
    snip_edges=False frames the half-sample-reflected signal (kaldi.py:44-83); round_to_power_of_two=False runs an FFT of
    the window's own length; subtract_mean needs nothing: AudioFeaturizer.forward subtracts the column mean again right
    after it, so the reference's result differs from plain CMN by rounding only."""

    def __init__(self, **kwargs):
        for k in kwargs:
            if k not in _FBANK_DEFAULTS:
                raise TypeError(f"fbank() got an unexpected keyword argument '{k}'")
        a = dict(_FBANK_DEFAULTS)
        a.update(kwargs)
        self.kwargs = kwargs
        sf = a['sample_frequency']
        self.hop = int(sf * a['frame_shift'] * 0.001)
        self.win_length = int(sf * a['frame_length'] * 0.001)
        if a['round_to_power_of_two']:
            self.n_fft = 1 if self.win_length == 0 else 2 ** (self.win_length - 1).bit_length()
        else:
            self.n_fft = self.win_length
        bad = []
        if a['dither'] != 0.0:
            bad.append(f"dither={a['dither']} (the reference draws fresh random noise on every call)")
        if a['min_duration'] != 0.0:
            bad.append(f"min_duration={a['min_duration']} (the reference returns an empty tensor for a shorter "
                       "utterance, which its torch.stack of the batch cannot take)")
        if a['channel'] not in (-1, 0):
            bad.append(f"channel={a['channel']} (the reference passes one mono row per utterance)")
        if a['use_energy']:
            bad.append('use_energy=True (the energy column is not counted by feature_dim, so no model consumes it; '
                       'raw_energy, energy_floor and htk_compat act only with it)')
        if not a['round_to_power_of_two'] and not _fft_size_ok(self.n_fft):
            bad.append(f'round_to_power_of_two=False with a {self.win_length}-sample window ({_FFT_SIZES})')
        _unsupported('Fbank', bad)
        self.n_mels = a['num_mel_bins']
        assert self.n_mels > 3, 'Must have at least 3 mel bins'
        wt = a['window_type']
        n = self.win_length
        if wt == 'povey':
            win = torch.hann_window(n, periodic=False, dtype=torch.float32).pow(0.85)
        elif wt == 'hanning':
            win = torch.hann_window(n, periodic=False, dtype=torch.float32)
        elif wt == 'hamming':
            win = torch.hamming_window(n, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float32)
        elif wt == 'rectangular':
            win = torch.ones(n, dtype=torch.float32)
        elif wt == 'blackman':
            c = 2 * math.pi / (n - 1)
            i = torch.arange(n, dtype=torch.float32)
            win = a['blackman_coeff'] - 0.5 * torch.cos(c * i) + (0.5 - a['blackman_coeff']) * torch.cos(2 * c * i)
        else:
            raise Exception('Invalid window type ' + wt)
        self.window = win.numpy().astype(np.float32)
        banks = kaldi_mel_banks(self.n_mels, self.n_fft, sf, a['low_freq'], a['high_freq'], a['vtln_low'],
                                a['vtln_high'], a['vtln_warp'])
        self.bank = _sparse_bank(banks.to(torch.float32).numpy())   # bin n_fft/2 has weight 0 (kaldi.py:627)
        self.desc = L.FrontendDesc(kind=0, n_fft=self.n_fft, win_length=self.win_length, hop=self.hop,
                                   n_mels=self.n_mels, remove_dc=1 if a['remove_dc_offset'] else 0,
                                   preemph=float(a['preemphasis_coefficient']), power=2 if a['use_power'] else 1,
                                   use_log=1 if a['use_log_fbank'] else 0, log_floor=float(np.finfo(np.float32).eps))
        self.opts = L.FrontendOptions(frame_mode=L.FRAME_DEFAULT if a['snip_edges'] else L.FRAME_KALDI_REFLECT, pad=0,
                                      spec_scale=1.0)


def _stft_args(defaults, name, kwargs):
    for k in kwargs:
        if k not in defaults and k not in ('window_fn', 'wkwargs'):
            raise TypeError(f"{name}.__init__() got an unexpected keyword argument '{k}'")
    a = dict(defaults)
    a.update(kwargs)
    n_fft = a['n_fft']
    win_length = a['win_length'] if a['win_length'] is not None else n_fft
    hop = a['hop_length'] if a['hop_length'] is not None else win_length // 2
    bad = []
    if a['power'] not in (1.0, 2.0, 1, 2):
        bad.append(f"power={a['power']} (|X| and |X|^2 are lowered)")
    if not _fft_size_ok(n_fft):
        bad.append(f'n_fft={n_fft} ({_FFT_SIZES})')
    if win_length > n_fft:
        bad.append(f'win_length={win_length} (longer than n_fft)')
    return a, n_fft, win_length, hop, bad


class MelSpectrogram:
    """kwargs of torchaudio.transforms.MelSpectrogram (featurizer.py:41-42): window_fn (periodic Hann by default), STFT
    framing of _stft_options, |X|^power, HTK or Slaney triangular bank (functional.py:518-587).  No log
    (featurizer.py:76)."""

    def __init__(self, **kwargs):
        a, n_fft, win_length, hop, bad = _stft_args(_MELSPEC_DEFAULTS, 'MelSpectrogram', kwargs)
        self.kwargs = kwargs
        f_max = a['f_max'] if a['f_max'] is not None else float(a['sample_rate'] // 2)
        if a['n_mels'] > n_fft // 2 + 1:
            bad.append(f"n_mels={a['n_mels']} (at most n_fft/2 + 1 = {n_fft // 2 + 1} filters)")
        _unsupported('MelSpectrogram', bad)
        self.n_fft, self.hop, self.n_mels = n_fft, hop, a['n_mels']
        self.window, taps = _stft_window(n_fft, win_length, kwargs.get('window_fn', torch.hann_window),
                                         kwargs.get('wkwargs'))
        self.opts = _stft_options(a, n_fft, taps)
        self.win_length = n_fft
        fb = melscale_fbanks(n_fft // 2 + 1, a['f_min'], f_max, self.n_mels, a['sample_rate'], a['norm'],
                             a['mel_scale'])
        self.bank = _sparse_bank(fb.T.contiguous().numpy())
        self.desc = L.FrontendDesc(kind=1, n_fft=n_fft, win_length=n_fft, hop=hop, n_mels=self.n_mels, remove_dc=0,
                                   preemph=0.0, power=int(a['power']), use_log=0, log_floor=0.0)
        self.dct = None
        self.n_out = self.n_mels


class Spectrogram:
    """kwargs of torchaudio.transforms.Spectrogram (featurizer.py:43-44): the MelSpectrogram pipeline without the mel
    projection -- the "bank" is the identity over the n_fft/2+1 bins, so the same kernel emits |X|^power directly."""

    def __init__(self, **kwargs):
        a, n_fft, win_length, hop, bad = _stft_args(_SPEC_DEFAULTS, 'Spectrogram', kwargs)
        self.kwargs = kwargs
        if not a['onesided']:
            bad.append('onesided=False (feature_dim counts n_fft/2 + 1 bins, so no model consumes the two-sided '
                       'spectrum)')
        _unsupported('Spectrogram', bad)
        nb = n_fft // 2 + 1
        self.n_fft, self.hop, self.n_mels = n_fft, hop, nb
        self.window, taps = _stft_window(n_fft, win_length, kwargs.get('window_fn', torch.hann_window),
                                         kwargs.get('wkwargs'))
        self.opts = _stft_options(a, n_fft, taps)
        self.win_length = n_fft
        idx = np.arange(nb, dtype=np.int32)
        self.bank = (idx, np.ones(nb, np.int32), idx.copy(), np.ones(nb, np.float32))
        self.desc = L.FrontendDesc(kind=1, n_fft=n_fft, win_length=n_fft, hop=hop, n_mels=nb, remove_dc=0, preemph=0.0,
                                   power=int(a['power']), use_log=0, log_floor=0.0)
        self.dct = None
        self.n_out = nb


class MFCC:
    """kwargs of torchaudio.transforms.MFCC (featurizer.py:45-46): MelSpectrogram(sample_rate, **melkwargs) ->
    AmplitudeToDB('power', top_db=80) (or log(mel + 1e-6) when log_mels) -> DCT-II (create_dct, functional.py:640-667)."""

    def __init__(self, **kwargs):
        for k in kwargs:
            if k not in _MFCC_DEFAULTS:
                raise TypeError(f"MFCC.__init__() got an unexpected keyword argument '{k}'")
        a = dict(_MFCC_DEFAULTS)
        a.update(kwargs)
        self.kwargs = kwargs
        if a['dct_type'] != 2:
            raise ValueError('DCT type not supported: {}'.format(a['dct_type']))
        mel = MelSpectrogram(sample_rate=a['sample_rate'], **(a['melkwargs'] or {}))
        n_mfcc, n_mels = a['n_mfcc'], mel.n_mels
        if n_mfcc > n_mels:
            raise ValueError('Cannot select more MFCC coefficients than # mel bins')
        _unsupported('MFCC', [f'n_mels={n_mels} (the DCT stage keeps its matrix in shared memory: at most 128 mel '
                              'bins)'] if n_mels > 128 else [])
        self.n_fft, self.hop, self.n_mels, self.win_length = mel.n_fft, mel.hop, n_mels, mel.win_length
        self.window, self.bank, self.opts = mel.window, mel.bank, mel.opts
        n = torch.arange(float(n_mels))
        k = torch.arange(float(n_mfcc)).unsqueeze(1)
        dct = torch.cos(math.pi / float(n_mels) * (n + 0.5) * k)
        if a['norm'] is None:
            dct *= 2.0
        else:
            assert a['norm'] == 'ortho'
            dct[0] *= 1.0 / math.sqrt(2.0)
            dct *= math.sqrt(2.0 / float(n_mels))
        self.dct = np.ascontiguousarray(dct.t().numpy(), dtype=np.float32)          # [n_mels, n_mfcc]
        self.n_out = n_mfcc
        if a['log_mels']:
            self.desc = L.FrontendDesc(kind=1, n_fft=mel.n_fft, win_length=mel.n_fft, hop=mel.hop, n_mels=n_mels,
                                       remove_dc=0, preemph=0.0, power=mel.desc.power, use_log=3, log_floor=1e-6,
                                       post=1, n_out=n_mfcc, db_mult=0.0, top_db=-1.0)
        else:
            self.desc = L.FrontendDesc(kind=1, n_fft=mel.n_fft, win_length=mel.n_fft, hop=mel.hop, n_mels=n_mels,
                                       remove_dc=0, preemph=0.0, power=mel.desc.power, use_log=2, log_floor=1e-10,
                                       post=1, n_out=n_mfcc, db_mult=10.0, top_db=80.0)


class HfFrontend:
    """`use_hf_model`: the wav2vec 2.0 / WavLM checkpoint named by `feature_method` (a local directory or a hub id
    already in the local cache, hf_checkpoint.resolve), lowered to the library's HF front-end (vp_frontend_set_hf):
    processor normalisation, conv feature encoder, feature projection LayerNorm -- everything `extract_features`
    depends on (featurizer.py:65-73).  `method_args['use_gpu']` is accepted and ignored, as on the reference's GPU."""

    def __init__(self, name, method_args):
        from .hf_checkpoint import HfCheckpoint
        self.ckpt = HfCheckpoint(name)
        c = self.ckpt
        n = len(c.conv_dim)
        if n > L.HF_MAX_LAYERS:
            raise NotImplementedError(f'{n} conv layers: the HF front-end runs at most {L.HF_MAX_LAYERS}')
        pad = lambda v: (C.c_int32 * L.HF_MAX_LAYERS)(*(list(v) + [0] * (L.HF_MAX_LAYERS - n)))
        self.hf_desc = L.HfDesc(n_layers=n, conv_dim=pad(c.conv_dim), conv_kernel=pad(c.conv_kernel),
                                conv_stride=pad(c.conv_stride), conv_bias=int(c.conv_bias),
                                norm=L.HF_NORM_GROUP if c.norm == 'group' else L.HF_NORM_LAYER,
                                do_normalize=int(c.do_normalize), norm_eps=1e-5, proj_eps=c.layer_norm_eps)
        self.n_mels = max(c.conv_dim)
        self.desc = L.FrontendDesc(kind=2, post=0, top_db=-1.0)     # what the featurizer asks of every front-end


class AudioFeaturizer:
    """音频特征器 (drop-in for mvector.data_utils.featurizer.AudioFeaturizer).

    :param feature_method: 'Fbank' | 'MelSpectrogram' | 'Spectrogram' | 'MFCC', or with use_hf_model a wav2vec 2.0 /
        WavLM checkpoint (local directory or cached hub id, HfFrontend)
    :param method_args: forwarded as **kwargs exactly like the reference (unknown keys -> TypeError)
    """

    def __init__(self, feature_method='MelSpectrogram', use_hf_model=False, method_args={}, engine=None):
        self._method_args = method_args
        self._feature_method = feature_method
        self.use_hf_model = use_hf_model
        if use_hf_model:
            self.feat_fun = HfFrontend(feature_method, method_args)
        elif feature_method == 'MelSpectrogram':
            self.feat_fun = MelSpectrogram(**method_args)
        elif feature_method == 'Fbank':
            self.feat_fun = KaldiFbank(**method_args)
        elif feature_method == 'Spectrogram':
            self.feat_fun = Spectrogram(**method_args)
        elif feature_method == 'MFCC':
            self.feat_fun = MFCC(**method_args)
        else:
            raise Exception(f'预处理方法 {self._feature_method} 不存在!')
        self.whole_call = self.feat_fun.desc.post == 1 and self.feat_fun.desc.top_db >= 0    # MFCC's call-wide clamp
        self._engine = engine
        self._configured = False
        if use_hf_model:
            logger.info(f'使用模型【{feature_method}】提取特征，使用【cuda】设备提取')
        else:
            logger.info(f'使用【{feature_method}】提取特征')

    # -- lazy device state so that constructing the object (config parsing) needs no GPU --
    def _ensure(self):
        if self._configured:
            return
        if self._engine is None:
            self._engine = Engine()
        f = self.feat_fun
        if self.use_hf_model:
            self._set_hf(f)
            self._configured = True
            return
        start, count, off, w = f.bank
        win = np.ascontiguousarray(f.window, dtype=np.float32)
        dct = getattr(f, 'dct', None)
        _check(self._engine.handle, L.lib().vp_frontend_set(
            self._engine.handle, C.byref(f.desc), win.ctypes.data_as(C.c_void_p), start.ctypes.data_as(C.c_void_p),
            count.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), w.ctypes.data_as(C.c_void_p), int(w.size),
            dct.ctypes.data_as(C.c_void_p) if dct is not None else C.c_void_p()))
        _check(self._engine.handle, L.lib().vp_frontend_set_options(self._engine.handle, C.byref(f.opts)))
        self._configured = True

    def _set_hf(self, f):
        c = f.ckpt
        n, wt = len(c.conv_dim), c.weights
        keep = []                                        # the host arrays stay alive until the library has copied them

        def ptrs(names):
            arr = (C.c_void_p * L.HF_MAX_LAYERS)()
            for i, k in enumerate(names):
                if k in wt:
                    a = np.ascontiguousarray(wt[k], dtype=np.float32)
                    keep.append(a)
                    arr[i] = a.ctypes.data
            return arr
        cw = ptrs([f'feature_extractor.conv_layers.{i}.conv.weight' for i in range(n)])
        cb = ptrs([f'feature_extractor.conv_layers.{i}.conv.bias' for i in range(n)])
        nw = ptrs([f'feature_extractor.conv_layers.{i}.layer_norm.weight' for i in range(n)])
        nb = ptrs([f'feature_extractor.conv_layers.{i}.layer_norm.bias' for i in range(n)])
        pw = np.ascontiguousarray(wt['feature_projection.layer_norm.weight'], dtype=np.float32)
        pb = np.ascontiguousarray(wt['feature_projection.layer_norm.bias'], dtype=np.float32)
        pp = C.POINTER(C.c_void_p)
        _check(self._engine.handle, L.lib().vp_frontend_set_hf(
            self._engine.handle, C.byref(f.hf_desc), C.cast(cw, pp), C.cast(cb, pp), C.cast(nw, pp), C.cast(nb, pp),
            pw.ctypes.data_as(C.c_void_p), pb.ctypes.data_as(C.c_void_p)))

    @property
    def engine(self):
        self._ensure()
        return self._engine

    def num_frames(self, n_samples):
        """Frames T for a waveform of n_samples (vp_num_frames): kaldi._get_strided, or torch.stft of the `pad`-extended
        signal, centred or not."""
        f = self.feat_fun
        if self.use_hf_model:
            return f.ckpt.num_frames(n_samples)
        mode = f.opts.frame_mode
        if f.desc.kind == 0:
            if mode == L.FRAME_KALDI_REFLECT:
                return (n_samples + f.hop // 2) // f.hop
            return 0 if n_samples < f.win_length else 1 + (n_samples - f.win_length) // f.hop
        n = n_samples + 2 * f.opts.pad
        if mode == L.FRAME_STFT_NOCENTER:
            return 0 if n < f.n_fft else 1 + (n - f.n_fft) // f.hop
        return 1 + n // f.hop

    def call_frames(self, n_samples):
        """num_frames of a padded call, which refuses a Kaldi window longer than its rows as the reference does."""
        f = self.feat_fun
        if f.desc.kind == 0:                            # kaldi.py:141
            assert 2 <= f.win_length <= n_samples, f'choose a window size {f.win_length} that is [2, {n_samples}]'
        return self.num_frames(n_samples)

    @staticmethod
    def keep_frames(input_lens_ratio, T):
        """featurizer.py:82-84: mask_lens = round(ratio * T) in float32, half-to-even."""
        r = torch.as_tensor(input_lens_ratio, dtype=torch.float32).cpu()
        return torch.round(r * T).to(torch.int32)

    def forward(self, waveforms, input_lens_ratio=None, group=None):
        """waveforms [B, L] (or [L]) float32 (torch CPU/CUDA tensor or ndarray) -> CUDA tensor [B, T, F].

        ``group``: a torch.distributed process group over which ONE reference call is sharded by utterances (every rank
        passes its shard, padded to the global longest item): only MFCC has a cross-utterance term -- the top_db clamp
        against the maximum of the whole call -- which is then all-reduced (MAX) between the mel stage and the DCT."""
        self._ensure()
        dev = self._engine.device
        w = torch.as_tensor(waveforms)
        if w.dim() == 1:
            w = w.unsqueeze(0)
        w = w.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
        B, Lp = w.shape
        T = self.num_frames(Lp)
        keep = None
        if input_lens_ratio is not None:
            keep = self.keep_frames(input_lens_ratio, T).to(dev, non_blocking=True)
        return self.forward_keep(w, keep, group=group)

    def forward_keep(self, w, keep=None, group=None):
        """Same with the mask lengths already on the device: ``w`` CUDA float32 [B, L] contiguous, ``keep`` CUDA int32 [B]
        (frames kept per utterance, featurizer.py:82-84) or None."""
        B, Lp = w.shape
        feats = torch.empty(B, self.num_frames(Lp), self.feature_dim, dtype=torch.float32, device=w.device)
        self.launch(w, feats, torch.cuda.current_stream(w.device), keep, group)
        return feats

    def launch(self, w, feats, stream, keep=None, group=None):
        """Enqueue vp_features on ``stream`` into ``feats``, a contiguous view of B * T * F floats (``w``, ``keep`` as for
        forward_keep).  ``group`` shards ONE call by utterances: MFCC then all-reduces (MAX) its clamp maximum between
        vp_mfcc_mel and vp_mfcc_finish, bit-identical to vp_features on the whole batch."""
        self._ensure()
        B, Lp = w.shape
        assert feats.is_contiguous() and feats.numel() == B * self.call_frames(Lp) * self.feature_dim
        lib, h = L.lib(), self._engine.handle
        wp, fp, sp = C.c_void_p(w.data_ptr()), C.c_void_p(feats.data_ptr()), C.c_void_p(stream.cuda_stream)
        kp = C.c_void_p(keep.data_ptr()) if keep is not None else C.c_void_p()
        with torch.cuda.stream(stream):
            scratch = torch.empty(max(int(lib.vp_frontend_scratch_floats(h, B, Lp)), 1), dtype=torch.float32,
                                  device=w.device)
            sc = C.c_void_p(scratch.data_ptr())
            if group is None or not self.whole_call:
                _check(h, lib.vp_features(h, wp, B, Lp, kp, fp, sc, sp))
                return
            import torch.distributed as dist
            mx = torch.empty(1, dtype=torch.float32, device=w.device)
            _check(h, lib.vp_mfcc_mel(h, wp, B, Lp, sc, C.c_void_p(mx.data_ptr()), sp))
            if dist.is_initialized() and dist.get_world_size(group) > 1:
                from ..distributed import device_collectives
                if device_collectives(group):
                    dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=group)
                else:                                   # gloo: one float through the host
                    m = mx.cpu()
                    dist.all_reduce(m, op=dist.ReduceOp.MAX, group=group)
                    mx.copy_(m)
            _check(h, lib.vp_mfcc_finish(h, B, Lp, kp, fp, sc, C.c_void_p(mx.data_ptr()), sp))

    def forward_each(self, w, lens):
        """Every row of a ragged batch featurized as if it were the whole call (vp_features_each): the reference's
        eval / feature-extraction mode, where each file is featurized alone (reader.py:82-107) and the features are then
        zero-padded to the longest (collate_fn.py:5-24).  ``w`` CUDA float32 [B, ld] contiguous, row b holding ``lens[b]``
        samples (host ints).  -> (feats CUDA [B, T, F], T the longest row's frames, row b +0.0 past its own frames;
        T_b numpy int32 [B]).  A row the one-row call would refuse raises that call's error: forward_keep's
        AssertionError for a Kaldi row shorter than the window, the library's length error for an STFT row."""
        self._ensure()
        B, ld = w.shape
        lens = np.asarray(lens, dtype=np.int64).reshape(-1)
        assert lens.size == B and (lens >= 0).all() and (lens <= ld).all(), 'one length in [0, ld] per row'
        lib = L.lib()
        h = self._engine.handle
        # Every length rule of the library (window, padding, at least one frame) holds for all lengths from some minimum
        # up, so the shortest row is the one to check: the library's host-only plan query refuses it exactly when a
        # one-row call would, and that one-row call then raises its own error before any launch.
        short = int(np.argmin(lens))
        info = (C.c_int32 * 8)()
        if lib.vp_frontend_plan_info(h, 1, int(lens[short]), self.feat_fun.desc.post, info) != L.VP_OK:
            self.forward_keep(w[short:short + 1, :int(lens[short])].contiguous())
            raise RuntimeError(f'row {short} of {int(lens[short])} samples is refused by the front-end')
        tb = np.array([self.num_frames(n) for n in lens.tolist()], dtype=np.int32)
        T = int(tb.max())
        dev = self._engine.device
        feats = torch.empty(B, T, self.feature_dim, dtype=torch.float32, device=dev)
        # the call's own scratch: sized by the longest row, not by the stride
        scratch = torch.empty(max(int(lib.vp_frontend_scratch_floats(h, B, int(lens.max()))), 1), dtype=torch.float32,
                              device=dev)
        lens_dev = torch.from_numpy(lens.astype(np.int32)).to(dev, non_blocking=True)
        _check(h, lib.vp_features_each(h, C.c_void_p(w.data_ptr()), B, ld, C.c_void_p(lens_dev.data_ptr()), T,
                                       C.c_void_p(feats.data_ptr()), C.c_void_p(scratch.data_ptr()),
                                       self._engine.stream_ptr()))
        return feats, tb

    __call__ = forward

    @property
    def feature_dim(self):
        """featurizer.py:93-111 (the HF model's output channels: conv_dim[-1])."""
        if self.use_hf_model:
            return self.feat_fun.ckpt.feature_dim
        if self._feature_method == 'MelSpectrogram':
            return self._method_args.get('n_mels', 128)
        elif self._feature_method == 'Spectrogram':
            return self._method_args.get('n_fft', 400) // 2 + 1
        elif self._feature_method == 'MFCC':
            return self._method_args.get('n_mfcc', 40)
        elif self._feature_method == 'Fbank':
            return self._method_args.get('num_mel_bins', 23)
        raise Exception('没有{}预处理方法'.format(self._feature_method))
