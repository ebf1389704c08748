"""The fused front-end's FFT core on the device (run on an H100: python -m pytest tests -m gpu): every n_fft class the
kernel has an instantiation for (256, 512, 1024, 2048: register-resident passes) and the plan-driven mixed-radix path
(400, 480, 600) against an fp64 numpy spectrum of the same fp32 windowed frames; frame counts around the 16-frame tile
and the frames-per-CTA boundaries, B = 1 and ragged batches; the CMN mean and run-to-run / batch-composition
determinism."""
import numpy as np
import pytest
import torch

from oracle import frontend as ofe
from test_gpu_parity import FBANK_EXACT_TOL

pytestmark = pytest.mark.gpu

FBANK = dict(sample_frequency=16000, num_mel_bins=80)


def _fz(method, args):
    from mvector.data_utils.featurizer import AudioFeaturizer
    return AudioFeaturizer(method, method_args=args)


def _noise(B, L, seed):
    return torch.randn(B, L, generator=torch.Generator().manual_seed(seed)) * 0.1


def _tones(B, L, n_fft):
    """A pure tone between two bins plus one 30 dB weaker: the weak line and the leakage floor sit far below the row
    maximum, where an exchange that mixed up two points would show."""
    t = torch.arange(L, dtype=torch.float64)
    rows = []
    for b in range(B):
        f1, f2 = (17.3 + 3 * b) / n_fft, (61.7 + 5 * b) / n_fft
        rows.append(0.5 * torch.sin(2 * np.pi * f1 * t) + 0.5 * 10 ** (-30 / 20) * torch.sin(2 * np.pi * f2 * t + 0.3))
    return torch.stack(rows).float()


def _exact_power_spectrogram(x, n_fft, hop):
    """torchaudio Spectrogram (centre, reflect, periodic Hann, power 2) with the window product in fp32 as the kernel and
    the reference form it, and the rFFT and |.|^2 in fp64.  -> raw power [B, T, n_fft/2+1] (float64)."""
    win = torch.hann_window(n_fft)
    xp = torch.nn.functional.pad(x[:, None], (n_fft // 2, n_fft // 2), mode='reflect')[:, 0]
    frames = xp.unfold(1, n_fft, hop) * win                                   # fp32 product
    z = np.fft.rfft(frames.numpy().astype(np.float64), axis=-1)
    return z.real ** 2 + z.imag ** 2


@pytest.mark.parametrize('signal', ['noise', 'tones'])
@pytest.mark.parametrize('n_fft', [256, 512, 1024, 2048, 400, 480, 600])
def test_spectrogram_against_fp64_spectrum(n_fft, signal):
    hop = n_fft // 4
    B, L = 3, hop * 36 + 7                                                    # T = 37: odd last frame, 16 | T - 5
    x = _noise(B, L, n_fft) if signal == 'noise' else _tones(B, L, n_fft)
    ratio = torch.tensor([1.0, 0.6, 0.31])
    got = _fz('Spectrogram', dict(n_fft=n_fft, hop_length=hop))(x, ratio).cpu().numpy().astype(np.float64)
    raw = _exact_power_spectrogram(x, n_fft, hop)
    T = raw.shape[1]
    assert got.shape == raw.shape == (B, T, n_fft // 2 + 1) and T == 37
    ref = raw.astype(np.float32).astype(np.float64)
    ref = ref - ref.mean(axis=1, keepdims=True)
    keep = torch.round(ratio * T).long().tolist()
    for b in range(B):
        row_max = raw[b].max(axis=1, keepdims=True)                           # per frame
        err = np.abs(got[b, :keep[b]] - ref[b, :keep[b]]) / row_max[:keep[b]]
        assert err.max() <= 2e-6, (n_fft, signal, b, err.max())
        assert np.all(got[b, keep[b]:] == 0)


# frames: one, one pair, around one 16-frame tile, around two and four tiles (the CTA sizes), and odd counts beyond
@pytest.mark.parametrize('T', [1, 2, 15, 16, 17, 31, 32, 33, 49, 63, 64, 65, 67, 130])
def test_fbank_frame_counts(T):
    L = 400 + 160 * (T - 1) + 3
    x = _noise(1, L, T)
    fz = _fz('Fbank', FBANK)
    got = fz(x).cpu()
    assert got.shape == (1, T, 80)
    exact = ofe.featurize(x, None, 'Fbank', FBANK, exact_spectrum=True)
    assert float((got - exact).abs().max()) <= FBANK_EXACT_TOL
    assert torch.equal(got, fz(x).cpu())


@pytest.mark.parametrize('method,args', [
    ('Fbank', FBANK),
    ('MelSpectrogram', dict(sample_rate=16000, n_fft=1024, win_length=1024, hop_length=320, f_min=50.0, f_max=14000.0,
                            n_mels=64)),
    ('Spectrogram', dict()),
    ('MFCC', dict()),
], ids=['Fbank', 'MelSpectrogram', 'Spectrogram', 'MFCC'])
def test_ragged_batch_cmn_and_determinism(method, args):
    B, L = 5, 16000 + 1234
    x = _noise(B, L, 7)
    ratio = torch.tensor([1.0, 0.93, 0.5, 0.07, 0.01])
    fz = _fz(method, args)
    got = fz(x, ratio).cpu()
    assert torch.equal(got, fz(x, ratio).cpu())                               # fixed summation orders, no atomics
    ref = ofe.featurize(x, ratio, method, args)
    tol = FBANK_EXACT_TOL if method == 'Fbank' else (2e-5 if method == 'MFCC' else 3e-6) * float(ref.abs().max())
    if method == 'Fbank':
        ref = ofe.featurize(x, ratio, method, args, exact_spectrum=True)
    assert float((got - ref).abs().max()) <= tol
    T = got.shape[1]
    keep = torch.round(ratio * T).long().tolist()
    for b in range(B):
        assert torch.all(got[b, keep[b]:] == 0)
    # the mean that was subtracted is the mean over ALL T frames: the unmasked utterance sums to ~0 per column
    full = fz(x[:1]).cpu()[0].double()
    scale = float(ofe.featurize(x[:1], None, method, args).abs().max())
    assert float(full.mean(0).abs().max()) <= 1e-5 * max(scale, 1.0)
    if method != 'MFCC':                      # MFCC's top_db clamp takes its maximum over the whole call
        assert torch.equal(full.float(), got[0])                              # an utterance does not see its batch
