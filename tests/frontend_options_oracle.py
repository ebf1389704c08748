"""CPU oracle of the front-end options beyond oracle/frontend.py's subset, torch fp32 like the reference (test
infrastructure, no torchaudio).  Restates, in this repository's own words:
  * kaldi.fbank with snip_edges=False (kaldi._get_strided: half-sample-symmetric reflection at both ends),
    round_to_power_of_two=False, VTLN-warped banks and subtract_mean            (kaldi.py:44-83, 436-511, 514-645)
  * torchaudio's spectrogram with `pad`, center=False, the four pad modes, `normalized` and window_fn
                                                                              (functional.py:52-144)
  * MelSpectrogram with the Slaney scale / norm, MFCC over it                 (functional.py:518-587, MFCC.forward)
The mel banks are the featurizer's host constants, which tests/test_frontend_options_cpu.py checks against torchaudio
on their own; everything else (framing, FFT, power, projection, log, CMN) is torch on the CPU."""
import torch

from oracle import frontend as ofe


def kaldi_frames(w, size, shift, snip_edges):
    """kaldi._get_strided: [m, size] frames of w."""
    L = w.numel()
    if snip_edges:
        m = ofe.num_frames(L, size, shift)
        return w.as_strided((m, size), (shift, 1))
    m = (L + shift // 2) // shift
    pad = size // 2 - shift // 2
    rev = torch.flip(w, [0])
    ext = torch.cat((rev[-pad:], w, rev)) if pad > 0 else torch.cat((w[-pad:], rev))
    return ext.as_strided((m, size), (shift, 1))


def kaldi_fbank(waveform, exact_spectrum=False, **kwargs):
    """One utterance -> [m, num_mel_bins]; ``exact_spectrum`` as in oracle.frontend.kaldi_fbank (fp64 FFT, power and
    projection on the same fp32 frames)."""
    from mvector.data_utils.featurizer import kaldi_mel_banks
    a = ofe.fbank_args(**kwargs)
    if a['dither'] != 0.0 or a['use_energy'] or a['min_duration'] != 0.0:
        raise NotImplementedError('oracle fbank: unsupported option')
    w = torch.as_tensor(waveform, dtype=torch.float32)
    shift, size, padded = ofe.frame_geometry(a['sample_frequency'], a['frame_shift'], a['frame_length'],
                                             a['round_to_power_of_two'])
    assert 2 <= size <= w.numel()
    frames = kaldi_frames(w, size, shift, a['snip_edges'])
    if a['remove_dc_offset']:
        frames = frames - frames.mean(dim=1, keepdim=True)
    c = a['preemphasis_coefficient']
    if c != 0.0:
        frames = frames - c * torch.cat([frames[:, :1], frames[:, :-1]], dim=1)
    frames = frames * ofe.feature_window(a['window_type'], size, a['blackman_coeff']).unsqueeze(0)
    if padded != size:
        frames = torch.nn.functional.pad(frames, (0, padded - size))
    banks = kaldi_mel_banks(a['num_mel_bins'], padded, a['sample_frequency'], a['low_freq'], a['high_freq'],
                            a['vtln_low'], a['vtln_high'], a['vtln_warp'])
    banks = torch.nn.functional.pad(banks.to(torch.float32), (0, 1))
    if exact_spectrum:
        spec = torch.fft.rfft(frames.double()).abs()
        spec = spec.pow(2.0) if a['use_power'] else spec
        mel = torch.mm(spec, banks.double().T).float()
    else:
        spec = torch.fft.rfft(frames).abs()
        spec = spec.pow(2.0) if a['use_power'] else spec
        mel = torch.mm(spec, banks.T)
    if a['use_log_fbank']:
        mel = torch.max(mel, torch.tensor(ofe.F32_EPS)).log()
    if a['subtract_mean']:
        mel = mel - mel.mean(dim=0, keepdim=True)
    return mel


def _stft_setup(a):
    n_fft = a['n_fft']
    win = a['win_length'] if a['win_length'] is not None else n_fft
    hop = a['hop_length'] if a['hop_length'] is not None else win // 2
    fn = a.get('window_fn', torch.hann_window)
    window = fn(win) if a.get('wkwargs') is None else fn(win, **a['wkwargs'])
    return n_fft, win, hop, window


def power_spectrogram(w, a):
    """functional.spectrogram: [B, L] -> [B, n_fft//2+1, T] |X|^power."""
    n_fft, win, hop, window = _stft_setup(a)
    w = torch.as_tensor(w, dtype=torch.float32)
    if a['pad'] > 0:
        w = torch.nn.functional.pad(w, (a['pad'], a['pad']), 'constant')
    norm = a['normalized']
    spec = torch.stft(w, n_fft=n_fft, hop_length=hop, win_length=win, window=window, center=a['center'],
                      pad_mode=a['pad_mode'], normalized=norm == 'frame_length', onesided=True, return_complex=True)
    if norm is True or norm == 'window':
        spec /= window.pow(2.0).sum().sqrt()
    return spec.abs() if a['power'] == 1.0 else spec.abs().pow(a['power'])


def mel_spectrogram(w, **kwargs):
    from mvector.data_utils.featurizer import melscale_fbanks
    a = dict(ofe._MELSPEC_KEYS)
    a.update(kwargs)
    spec = power_spectrogram(w, a)
    f_max = a['f_max'] if a['f_max'] is not None else float(a['sample_rate'] // 2)
    fb = melscale_fbanks(a['n_fft'] // 2 + 1, a['f_min'], f_max, a['n_mels'], a['sample_rate'], a['norm'],
                         a['mel_scale'])
    return torch.matmul(spec.transpose(-1, -2), fb).transpose(-1, -2)


def spectrogram(w, **kwargs):
    a = dict(ofe._SPEC_KEYS)
    a.update(kwargs)
    return power_spectrogram(w, a)


def mfcc(w, **kwargs):
    a = dict(ofe._MFCC_KEYS)
    a.update(kwargs)
    mel = mel_spectrogram(w, sample_rate=a['sample_rate'], **(a['melkwargs'] or {}))
    mel = torch.log(mel + 1e-6) if a['log_mels'] else ofe.power_to_db(mel)
    return torch.matmul(mel.transpose(-1, -2), ofe.dct_matrix(a['n_mfcc'], mel.shape[-2], a['norm'])).transpose(-1, -2)


def featurize(waveforms, input_lens_ratio=None, feature_method='Fbank', method_args=None, exact_spectrum=False):
    """AudioFeaturizer.forward (featurizer.py:53-91) over the option-aware transforms: [B, T, F] float32."""
    args = dict(method_args or {})
    w = torch.as_tensor(waveforms, dtype=torch.float32)
    if w.dim() == 1:
        w = w.unsqueeze(0)
    if feature_method == 'Fbank':
        feat = torch.stack([kaldi_fbank(x, exact_spectrum=exact_spectrum, **args).transpose(0, 1) for x in w])
    else:
        feat = {'MelSpectrogram': mel_spectrogram, 'Spectrogram': spectrogram, 'MFCC': mfcc}[feature_method](w, **args)
    feat = feat.transpose(2, 1)
    feat = feat - feat.mean(1, keepdim=True)
    if input_lens_ratio is not None:
        keep = torch.round(torch.as_tensor(input_lens_ratio, dtype=torch.float32) * feat.shape[1]).long().unsqueeze(1)
        idx = torch.arange(feat.shape[1]).repeat(feat.shape[0], 1)
        feat = torch.where((idx < keep).unsqueeze(-1), feat, torch.zeros_like(feat))
    return feat
