"""Generate tests/golden/frontend_options.npz: outputs of the UNMODIFIED reference's AudioFeaturizer on the front-end
options beyond the shipped configurations (snip_edges=False, round_to_power_of_two=False, VTLN, subtract_mean,
center=False, the four pad modes, pad, normalized, window_fn, the Slaney mel scale and norm, n_mels above 128, and
combinations), for tests/test_frontend_options_cpu.py to pin the options oracle against.

    python tests/golden/make_frontend_options_golden.py      (needs the reference checkout make_golden.py points at)

Each case runs a ragged batch (zero-padded to the longest item, with length ratios) and a single utterance; as in
full_size_reference.npz only the shape, a fixed seeded sample of the values and the float64 sum are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))

_FB = dict(sample_frequency=16000, num_mel_bins=80)
_MEL = dict(sample_rate=16000, n_fft=512, win_length=400, hop_length=160, n_mels=64)
CASES = [
    ('Fbank', dict(_FB, snip_edges=False)),
    ('Fbank', dict(_FB, round_to_power_of_two=False)),
    ('Fbank', dict(_FB, vtln_warp=0.9)),
    ('Fbank', dict(_FB, subtract_mean=True)),
    ('Fbank', dict(_FB, snip_edges=False, round_to_power_of_two=False)),
    ('Fbank', dict(sample_frequency=8000, num_mel_bins=40, snip_edges=False, round_to_power_of_two=False,
                   vtln_warp=1.1, window_type='hamming')),
    ('MelSpectrogram', dict(_MEL, center=False)),
    ('MelSpectrogram', dict(_MEL, pad_mode='constant')),
    ('MelSpectrogram', dict(_MEL, pad_mode='replicate')),
    ('MelSpectrogram', dict(_MEL, pad_mode='circular')),
    ('MelSpectrogram', dict(_MEL, pad=100)),
    ('MelSpectrogram', dict(_MEL, normalized=True)),
    ('MelSpectrogram', dict(_MEL, normalized='frame_length')),
    ('MelSpectrogram', dict(_MEL, norm='slaney', mel_scale='slaney')),
    ('MelSpectrogram', dict(sample_rate=16000, n_fft=1024, hop_length=320, n_mels=200)),
    ('MelSpectrogram', dict(_MEL, center=False, norm='slaney', mel_scale='slaney', normalized=True)),
    ('MelSpectrogram', dict(_MEL, window_fn=torch.hamming_window, wkwargs=dict(periodic=False))),
    ('MelSpectrogram', dict(_MEL, pad=40, pad_mode='circular', power=1.0)),
    ('Spectrogram', dict(center=False, normalized='window')),
    ('Spectrogram', dict(n_fft=512, hop_length=160, pad=40, pad_mode='replicate', normalized='frame_length')),
    ('MFCC', dict(n_mfcc=24, melkwargs=dict(n_fft=512, hop_length=160, n_mels=64, center=False, norm='slaney',
                                            mel_scale='slaney'))),
    ('MFCC', dict(log_mels=True, melkwargs=dict(n_fft=400, pad_mode='constant', normalized=True, n_mels=64))),
]
LENS = (16000, 12611, 6403)
N_SAMPLE = 384


def front_input():
    """Seeded ragged batch (zero-padded, length ratios) and its second utterance alone."""
    g = torch.Generator().manual_seed(21)
    waves = [(torch.randn(n, generator=g) * 0.1).numpy() for n in LENS]
    lmax = max(LENS)
    x = np.zeros((len(waves), lmax), dtype=np.float32)
    for i, w in enumerate(waves):
        x[i, :len(w)] = w
    ratio = np.asarray([n / lmax for n in LENS], dtype=np.float32)
    return torch.from_numpy(x), torch.from_numpy(ratio), torch.from_numpy(waves[1])


def sample_index(n, key):
    rng = np.random.default_rng(2000 + key)
    return np.sort(rng.choice(n, size=min(n, N_SAMPLE), replace=False))


def main():
    sys.path.insert(0, HERE)
    from make_golden import ROOT, install_yeaudio_stub       # puts the reference checkout first on sys.path
    install_yeaudio_stub()
    from loguru import logger
    logger.remove()
    from mvector.data_utils.featurizer import AudioFeaturizer  # reference
    assert not os.path.abspath(sys.modules['mvector'].__file__).startswith(ROOT + os.sep), 'not the reference'
    x, ratio, one = front_input()
    out = {}
    for i, (method, args) in enumerate(CASES):
        fz = AudioFeaturizer(method, method_args=args)
        for tag, y in (('batch', fz(x, ratio)), ('single', fz(one))):
            y = y.numpy()
            out[f'case{i}/{tag}/shape'] = np.array(y.shape, dtype=np.int64)
            out[f'case{i}/{tag}/sample'] = y.reshape(-1)[sample_index(y.size, 2 * i + (tag == 'single'))]
            out[f'case{i}/{tag}/sum'] = np.array(y.astype(np.float64).sum())
        out[f'case{i}/feature_dim'] = np.array(fz.feature_dim, dtype=np.int64)
        print(f'{method:14s} {str(args)[:90]} {tuple(y.shape)}')
    np.savez_compressed(os.path.join(HERE, 'frontend_options.npz'), **out)


if __name__ == '__main__':
    main()
