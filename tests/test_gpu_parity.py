"""GPU parity tests (run on an H100: python -m pytest tests -m gpu).  Everything goes through the C ABI
(libvpb200.so) and is compared with the CPU oracle, the reference's golden vectors and the numpy plan interpreter.
Tolerance: embeddings within 1e-4 relative L2 of the reference fp32 forward (BASELINE.json north_star)."""
import os
import tempfile
import wave

import numpy as np
import pytest
import torch

from conftest import load_golden, rel_l2

pytestmark = pytest.mark.gpu

EMB_TOL = 1e-4          # north_star: "within 1e-4 relative fp32"
# Log-mel parity (values span about [-16, +6]).  The reference's own fp32 FFT is up to ~6e-4 away from the exact value of
# its formula on white-noise input (pre-emphasis leaves the low bins 30 dB below the frame energy and the log turns their
# relative error into an absolute one; tools/fbank_precision_study.py), so |ours - reference| cannot be bounded below
# that by ANY implementation.  The front-end kernel therefore computes the spectrum in fp64 and the tests check
#   (1) |ours - exact| <= FBANK_EXACT_TOL   (exact = oracle with exact_spectrum=True: same fp32 frames, fp64 spectrum)
#   (2) |ours - reference| <= |reference - exact| + FBANK_EXACT_TOL   (never farther than the reference's own rounding)
# What is left of (1) is the per-frame DC mean: an fp32 sum of 400 samples whose summation order is
# implementation defined (torch's vectorised sum vs a warp butterfly here); its last-bit difference leaks into the
# lowest bins through the window.
FBANK_EXACT_TOL = 1e-4
FBANK_ABS_TOL = 2e-3    # hard cap on |ours - reference| whatever the input


def _fbank_three_way(got, waves, ratio, args):
    """-> (|ours - exact|, |ours - ref|, |ref - exact|) max-abs on CMN'd log-mel features."""
    from oracle import frontend as ofe
    ref = ofe.featurize(waves, ratio, 'Fbank', args)
    exact = ofe.featurize(waves, ratio, 'Fbank', args, exact_spectrum=True)
    assert got.shape == ref.shape
    e_got, e_ref, d = (got - exact).abs().max().item(), (ref - exact).abs().max().item(), (got - ref).abs().max().item()
    print(f'fbank: |ours-exact| {e_got:.2e}  |ours-ref| {d:.2e}  |ref-exact| {e_ref:.2e}')
    assert e_got <= FBANK_EXACT_TOL, (e_got, e_ref)
    assert d <= e_ref + FBANK_EXACT_TOL and d < FBANK_ABS_TOL, (d, e_ref)
    return e_got, d, e_ref


def _model(name, fdim, margs, sd, engine_pref=None):
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object
    m = build_model(fdim, dict_to_object({'model_conf': {'model': name, 'model_args': margs}}))
    m.load_state_dict({'0.' + k: v for k, v in sd.items()})
    if engine_pref is not None:
        m.engine_pref = engine_pref
    return m


def _featurizer(prep):
    from mvector.data_utils.featurizer import AudioFeaturizer
    return AudioFeaturizer(prep['feature_method'], method_args=prep['method_args'])


# ------------------------------------------------------------------------------------------------ front-end
@pytest.mark.parametrize('n', [400, 559, 560, 7999, 16000, 48000])
def test_fbank_single_lengths(n):
    from oracle import frontend as ofe
    args = dict(sample_frequency=16000, num_mel_bins=80)
    g = torch.Generator().manual_seed(n)
    w = torch.randn(2, n, generator=g) * 0.1
    fz = _featurizer(dict(feature_method='Fbank', method_args=args))
    got = fz(w).cpu()
    assert got.shape == (2, 1 + (n - 400) // 160, 80)
    _fbank_three_way(got, w, None, args)


def test_fbank_ragged_batch_semantics():
    """Reference ragged semantics (SURVEY.md 9.2): zero-pad to Lmax, CMN over ALL frames, frames >= round(ratio*T) = 0."""
    from oracle import frontend as ofe
    args = dict(sample_frequency=16000, num_mel_bins=80)
    g = torch.Generator().manual_seed(11)
    waves = [(torch.randn(n, generator=g) * 0.1).numpy() for n in (16000, 48000, 30001, 5000)]
    x, ratio = ofe.pad_batch(waves)
    ref = ofe.featurize(x, ratio, 'Fbank', args)
    fz = _featurizer(dict(feature_method='Fbank', method_args=args))
    got = fz(torch.from_numpy(x), torch.from_numpy(ratio)).cpu()
    _fbank_three_way(got, x, ratio, args)
    keep = torch.round(torch.from_numpy(ratio) * ref.shape[1]).long()
    for i, k in enumerate(keep.tolist()):
        assert torch.all(got[i, k:] == 0)          # masked frames are exactly zero
    # an all-zero (silent) utterance hits the log floor exactly like the reference
    z = torch.zeros(1, 8000)
    assert torch.equal(fz(z).cpu(), ofe.featurize(z, None, 'Fbank', args))


@pytest.mark.parametrize('margs', [
    dict(sample_rate=16000, n_fft=1024, win_length=1024, hop_length=320, f_min=50.0, f_max=14000.0, n_mels=64),
    dict(sample_rate=16000, n_fft=512, win_length=512, hop_length=160, f_min=50.0, f_max=7600.0, n_mels=16),
    dict(sample_rate=16000, n_fft=512, win_length=400, hop_length=200, n_mels=40),
])
def test_melspectrogram(margs):
    from oracle import frontend as ofe
    g = torch.Generator().manual_seed(5)
    waves = [(torch.randn(n, generator=g) * 0.1).numpy() for n in (16000, 12345)]
    x, ratio = ofe.pad_batch(waves)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref = ofe.featurize(x, ratio, 'MelSpectrogram', margs)
    fz = _featurizer(dict(feature_method='MelSpectrogram', method_args=margs))
    got = fz(torch.from_numpy(x), torch.from_numpy(ratio)).cpu()
    assert got.shape == ref.shape
    # raw power mel (no log, featurizer.py:76): compare relative to the dynamic range
    assert ((got - ref).abs().max() / ref.abs().max()).item() < 2e-6


@pytest.mark.parametrize('method,margs', [
    ('MelSpectrogram', dict()),                                              # torchaudio defaults: n_fft 400 (radix-5 passes)
    ('Spectrogram', dict()),                                                 # 201 pass-through bins
    ('Spectrogram', dict(n_fft=512, hop_length=160, power=1.0)),
    ('Spectrogram', dict(n_fft=480, win_length=400)),                        # radix-3 pass, short window centred in n_fft
])
def test_stft_frontends_mixed_radix(method, margs):
    """SURVEY.md 8(f): Spectrogram (featurizer.py:43-44) and non-power-of-two n_fft through the same fused kernel."""
    from oracle import frontend as ofe
    g = torch.Generator().manual_seed(6)
    waves = [(torch.randn(n, generator=g) * 0.1).numpy() for n in (16000, 12345, 4000)]
    x, ratio = ofe.pad_batch(waves)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref = ofe.featurize(x, ratio, method, margs)
    fz = _featurizer(dict(feature_method=method, method_args=margs))
    got = fz(torch.from_numpy(x), torch.from_numpy(ratio)).cpu()
    assert got.shape == ref.shape and got.shape[2] == fz.feature_dim
    assert ((got - ref).abs().max() / ref.abs().max()).item() < 3e-6
    one = fz(torch.from_numpy(waves[1])).cpu()
    ref1 = ofe.featurize(waves[1], None, method, margs)
    assert ((one - ref1).abs().max() / ref1.abs().max()).item() < 3e-6


@pytest.mark.parametrize('margs', [
    dict(),                                                                  # n_fft 400, 128 mels, 40 coefficients, top_db 80
    dict(n_mfcc=24, melkwargs=dict(n_fft=512, hop_length=160, n_mels=64, f_min=20.0)),
    dict(log_mels=True, norm=None, melkwargs=dict(n_fft=512, n_mels=40)),
])
def test_mfcc(margs):
    """torchaudio.transforms.MFCC (featurizer.py:45-46): dB with the call-wide top_db clamp (the quiet third utterance
    is clamped by the loud ones' maximum), DCT-II, then CMN + mask."""
    from oracle import frontend as ofe
    g = torch.Generator().manual_seed(7)
    waves = [(torch.randn(n, generator=g) * a).numpy() for n, a in ((16000, 0.1), (12345, 0.3), (9000, 1e-5))]
    x, ratio = ofe.pad_batch(waves)
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref = ofe.featurize(x, ratio, 'MFCC', margs)
        ref1 = ofe.featurize(waves[2], None, 'MFCC', margs)
    fz = _featurizer(dict(feature_method='MFCC', method_args=margs))
    got = fz(torch.from_numpy(x), torch.from_numpy(ratio)).cpu()
    assert got.shape == ref.shape
    assert ((got - ref).abs().max() / ref.abs().max()).item() < 2e-5
    one = fz(torch.from_numpy(waves[2])).cpu()                               # alone, the quiet utterance is NOT clamped
    assert ((one - ref1).abs().max() / ref1.abs().max()).item() < 2e-5


def test_frontend_loud_errors():
    from mvector._lib import VpError
    fz = _featurizer(dict(feature_method='Fbank', method_args=dict(sample_frequency=16000, num_mel_bins=80)))
    with pytest.raises(AssertionError):
        fz(torch.zeros(1, 300))                     # shorter than one frame: reference asserts too (kaldi.py:141)
    with pytest.raises(NotImplementedError):
        _featurizer(dict(feature_method='MelSpectrogram', method_args=dict(n_fft=442)))     # 2 * 13 * 17
    with pytest.raises(TypeError):
        _featurizer(dict(feature_method='Fbank', method_args=dict(n_mels=80)))
    assert VpError is not None


# ------------------------------------------------------------------------------------------------ backbones
SMALL = ['ecapa_small', 'tdnn_small', 'campplus_small', 'resnetse_small', 'eres2net_small', 'eres2net_wide_small',
         'ecapa_sap_small', 'tdnn_tsp_small', 'resnetse_tap_small', 'res2net_small', 'eres2netv2_small', 'tdnn_spec_small',
         'resnetse_mfcc_small', 'ecapa_mfcc400_small']


@pytest.mark.parametrize('name', SMALL)
def test_small_models_vs_reference_golden(name, manifest):
    """Backbone from the reference's golden FEATURES -> embedding, and waveform -> embedding through the fused path.
    The program runs three times on the same input and output tensors -- eager, captured as a CUDA graph, replayed --
    with bit-identical embeddings."""
    from plan_sim import simulate
    m = manifest[name]
    z, sd = load_golden(name)
    model = _model(m['model'], m['feature_dim'], m['model_args'], sd)
    feats = torch.from_numpy(z['feats']).cuda().float().contiguous()
    prog = model.program(feats.shape[0], feats.shape[1])
    y = torch.empty(feats.shape[0], model.embd_dim, device='cuda')
    runs = []
    for _ in range(3):
        y.fill_(float('nan'))
        prog.run(feats, y)
        runs.append(y.cpu().numpy())
    for label, r in zip(('captured', 'replayed'), runs[1:]):
        assert np.array_equal(r.view(np.uint32), runs[0].view(np.uint32)), label
    emb = runs[0]
    assert rel_l2(emb, z['emb']).max() < EMB_TOL
    sim, _ = simulate(model, z['feats'])
    assert rel_l2(emb, sim).max() < EMB_TOL
    # full path from waveforms (ragged batch, reference padding semantics)
    from oracle import frontend as ofe
    waves = [z['wave%d' % i] for i in range(len(m['lens']))]
    x, ratio = ofe.pad_batch(waves)
    fz = _featurizer(m['preprocess'])
    emb2 = model(fz(torch.from_numpy(x), torch.from_numpy(ratio))).cpu().numpy()
    assert rel_l2(emb2, z['emb']).max() < EMB_TOL
    emb1 = model(fz(torch.from_numpy(waves[-1]))).cpu().numpy()[0]
    assert rel_l2(emb1, z['emb_single_last']).max() < EMB_TOL


FULL = [
    ('EcapaTdnn', dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536]), 80, 3, 298),
    ('TDNN', dict(embd_dim=192, channels=512, pooling_type='ASP'), 80, 3, 218),
    ('CAMPPlus', dict(embd_dim=192), 80, 2, 298),
    ('ResNetSE', dict(embd_dim=192, pooling_type='ASP'), 64, 2, 151),
    ('ERes2Net', dict(embd_dim=192, m_channels=32), 80, 2, 130),
    ('ERes2Net', dict(embd_dim=192, m_channels=64, mul_channel=2, expansion=4, base_width=24, scale=3), 80, 1, 98),
    ('Res2Net', dict(embd_dim=192, pooling_type='ASP', m_channels=32), 80, 3, 298),
    ('ERes2NetV2', dict(embd_dim=192, m_channels=32), 80, 2, 130),
]


@pytest.mark.parametrize('model,margs,fdim,B,T', FULL, ids=[f[0] + str(i) for i, f in enumerate(FULL)])
def test_full_size_models_vs_oracle(model, margs, fdim, B, T):
    """BASELINE.json model configurations at full width, seeded weights, features ~ CMN'd log-mel statistics."""
    from oracle import models as om
    sd = om.random_state_dict(model, fdim, seed=3, gain=om.CONDITIONED_GAIN[model], **margs)
    g = torch.Generator().manual_seed(17)
    feats = torch.randn(B, T, fdim, generator=g) * 2.0
    ref = om.forward(model, sd, feats, **margs).numpy()
    got = _model(model, fdim, margs, sd)(feats.cuda()).cpu().numpy()
    assert rel_l2(got, ref).max() < EMB_TOL


def test_ecapa_intermediates_vs_plan_sim(manifest):
    """Per-block activations (tapped from the workspace) against the numpy interpreter: localises a failing kernel."""
    from plan_sim import Sim
    m = manifest['ecapa_small']
    z, sd = load_golden('ecapa_small')
    model = _model(m['model'], m['feature_dim'], m['model_args'], sd)
    feats = z['feats']
    B, T, _ = feats.shape
    prog = model.program(B, T)
    emb = torch.empty(B, model.embd_dim, device='cuda')
    prog.run(torch.from_numpy(feats).cuda().contiguous(), emb)
    pb = model.lower(B, T)
    s = Sim(pb, model._blob, feats)
    s.run()
    for name, (view, rows) in pb.taps.items():
        got = prog.peek(name).cpu().numpy()
        ref = s.rd(view.off, rows, view.ld, view.coff, view.C)
        err = np.abs(got - ref).max() / max(np.abs(ref).max(), 1e-9)
        assert err < 1e-5, (name, err)


# ------------------------------------------------------------------------------------------------ predictor
def _cfg(model, margs, prep, db_norm=False):
    return {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                         'use_dB_normalization': db_norm, 'target_dB': -20},
                             'eval_conf': {'batch_size': 16, 'max_duration': 20}},
            'preprocess_conf': {'use_hf_model': False, 'feature_method': prep['feature_method'],
                                'method_args': dict(prep['method_args'])},
            'model_conf': {'model': model, 'model_args': dict(margs)}}


def test_predictor_dropin_predict_batch(manifest):
    from mvector.predict import MVectorPredictor
    m = manifest['ecapa_small']
    z, sd = load_golden('ecapa_small')
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        pred = MVectorPredictor(configs=_cfg(m['model'], m['model_args'], m['preprocess']), model_path=td, use_gpu=True)
        with pytest.raises(AssertionError):
            MVectorPredictor(configs=_cfg(m['model'], m['model_args'], m['preprocess']),
                             model_path=os.path.join(td, 'nope'), use_gpu=True)
    waves = [z['wave%d' % i] for i in range(len(m['lens']))]
    emb = pred.predict_batch(waves)
    assert emb.shape == z['emb'].shape and emb.dtype == np.float32
    assert rel_l2(emb, z['emb']).max() < EMB_TOL
    e1 = pred.predict(waves[-1])
    assert rel_l2(e1, z['emb_single_last']).max() < EMB_TOL
    with pytest.raises(AssertionError):
        pred.predict(np.zeros(1000, dtype=np.float32))        # < min_duration (predict.py:204-205)
    with pytest.raises(Exception):
        pred.predict(12345)                                   # unsupported type (predict.py:203)
    with pytest.raises(RuntimeError):
        MVectorPredictor(configs=_cfg(m['model'], m['model_args'], m['preprocess']), model_path='x', use_gpu=False)


def test_c1_infer_contrast_flow(manifest):
    """BASELINE config #1: configs/tdnn.yml surface, dataset/a_1.wav vs a_2.wav (infer_contrast.py:19-23)."""
    from mvector.predict import MVectorPredictor
    from oracle import models as om
    m = manifest['c1_tdnn_contrast']
    z, _ = load_golden('c1_tdnn_contrast')
    sd = om.random_state_dict('TDNN', 80, seed=m['seed'], **m['model_args'])
    prep = dict(feature_method='Fbank', method_args=dict(sample_frequency=16000, num_mel_bins=80))
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        paths = []
        for nm in ('a_1', 'a_2'):
            p = os.path.join(td, nm + '.wav')
            with wave.open(p, 'wb') as w:
                w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000)
                w.writeframes(z['pcm_' + nm].astype('<i2').tobytes())
            paths.append(p)
        pred = MVectorPredictor(configs=_cfg('TDNN', m['model_args'], prep, db_norm=True), model_path=td, use_gpu=True)
        e1, e2 = pred.predict(paths[0]), pred.predict(paths[1])
        sim = float(pred.contrast(paths[0], paths[1]))
    assert rel_l2(e1, z['emb_a_1']).max() < EMB_TOL and rel_l2(e2, z['emb_a_2']).max() < EMB_TOL
    assert abs(sim - float(z['sim'])) < 1e-4


# ------------------------------------------------------------------------------------------------ full-size properties
def test_c2_full_batch_properties():
    """BASELINE config #2 (EcapaTdnn + Fbank, B=256 x 3 s): size-independent properties + sampled oracle check."""
    from oracle import frontend as ofe
    from oracle import models as om
    margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
    fargs = dict(sample_frequency=16000, num_mel_bins=80)
    sd = om.random_state_dict('EcapaTdnn', 80, seed=0, **margs)
    model = _model('EcapaTdnn', 80, margs, sd)
    fz = _featurizer(dict(feature_method='Fbank', method_args=fargs))
    g = torch.Generator().manual_seed(1236)
    wave_ = torch.randn(256, 48000, generator=g) * 0.1
    wd = wave_.cuda()
    e = model(fz(wd))
    e_again = model(fz(wd))
    assert torch.equal(e, e_again)                              # deterministic (no atomics on the path)
    perm = torch.randperm(256, generator=g)
    e_perm = model(fz(wd[perm.cuda()]))
    assert torch.equal(e_perm, e[perm.cuda()])                  # batch-permutation equivariance, bit exact
    e_small = model(fz(wd[:4]))
    assert rel_l2(e_small.cpu().numpy(), e[:4].cpu().numpy()).max() < 1e-5   # per-utterance independence
    idx = [0, 100, 255]
    ref = om.forward('EcapaTdnn', sd, ofe.featurize(wave_[idx], None, 'Fbank', fargs), **margs).numpy()
    assert rel_l2(e[idx].cpu().numpy(), ref).max() < EMB_TOL


# ------------------------------------------------------------------------------------------------ BASELINE configs 3-5
def _ragged(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(n, generator=g) * 0.1).numpy() for n in lens]


def test_c3_campplus_fbank_batch():
    """BASELINE config #3 (per-GPU shard shape, reduced batch): CAM++ + Fbank-80 on 3 s utterances, waveform -> embedding."""
    from oracle import frontend as ofe
    from oracle import models as om
    margs, fargs = dict(embd_dim=192), dict(sample_frequency=16000, num_mel_bins=80)
    sd = om.random_state_dict('CAMPPlus', 80, seed=5, **margs)
    waves = _ragged([48000] * 6, 31)
    x, ratio = ofe.pad_batch(waves)
    ref = om.forward('CAMPPlus', sd, ofe.featurize(x, ratio, 'Fbank', fargs), **margs).numpy()
    fz = _featurizer(dict(feature_method='Fbank', method_args=fargs))
    got = _model('CAMPPlus', 80, margs, sd)(fz(torch.from_numpy(x), torch.from_numpy(ratio))).cpu().numpy()
    assert rel_l2(got, ref).max() < EMB_TOL


def test_c4_resnetse_melspectrogram_5s():
    """BASELINE config #4: ResNetSE + MelSpectrogram (README.md:303-311 method_args; the shipped yml's Fbank args make
    MelSpectrogram(**args) raise TypeError, SURVEY.md finding 3), 5 s @ 16 kHz -> [B, 251, 64]."""
    import warnings
    from oracle import frontend as ofe
    from oracle import models as om
    fargs = dict(sample_rate=16000, n_fft=1024, win_length=1024, hop_length=320, f_min=50.0, f_max=14000.0, n_mels=64)
    margs = dict(embd_dim=192, pooling_type='ASP')
    sd = om.random_state_dict('ResNetSE', 64, seed=6, gain=om.CONDITIONED_GAIN['ResNetSE'], **margs)
    waves = _ragged([80000] * 3, 32)
    x, ratio = ofe.pad_batch(waves)
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        feats = ofe.featurize(x, ratio, 'MelSpectrogram', fargs)
        fz = _featurizer(dict(feature_method='MelSpectrogram', method_args=fargs))
    assert feats.shape == (3, 251, 64)
    # raw power mel features (no log) have a huge dynamic range; scale like a dB-normalised recording keeps them finite
    ref = om.forward('ResNetSE', sd, feats, **margs).numpy()
    got = _model('ResNetSE', 64, margs, sd)(fz(torch.from_numpy(x), torch.from_numpy(ratio))).cpu().numpy()
    assert rel_l2(got, ref).max() < EMB_TOL
    with pytest.raises(TypeError):                       # the shipped configs/resnet_se.yml method_args
        _featurizer(dict(feature_method='MelSpectrogram', method_args=dict(sample_frequency=16000, num_mel_bins=80)))


def test_c5_eres2net55m_ragged_1_to_10s():
    """BASELINE config #5: the 55.2 M ERes2Net (m_channels=64, mul_channel=2, expansion=4, base_width=24, scale=3) on a
    ragged 1-10 s batch padded to its max (reference ragged semantics: T from Lmax, masked frames are zeros)."""
    from oracle import frontend as ofe
    from oracle import models as om
    margs = dict(embd_dim=192, m_channels=64, mul_channel=2, expansion=4, base_width=24, scale=3)
    fargs = dict(sample_frequency=16000, num_mel_bins=80)
    sd = om.random_state_dict('ERes2Net', 80, seed=8, gain=om.CONDITIONED_GAIN['ERes2Net'], **margs)
    # 1 s and 10 s when VPB_SLOW_TESTS=1 (the CPU oracle needs minutes for 2 x 312 GFLOP); 1 s and 4 s by default
    long = 160000 if os.environ.get('VPB_SLOW_TESTS') else 64000
    waves = _ragged([16000, long], 33)
    x, ratio = ofe.pad_batch(waves)
    feats = ofe.featurize(x, ratio, 'Fbank', fargs)
    assert feats.shape == (2, 1 + (long - 400) // 160, 80)
    ref = om.forward('ERes2Net', sd, feats, **margs).numpy()
    fz = _featurizer(dict(feature_method='Fbank', method_args=fargs))
    got = _model('ERes2Net', 80, margs, sd)(fz(torch.from_numpy(x), torch.from_numpy(ratio))).cpu().numpy()
    assert rel_l2(got, ref).max() < EMB_TOL


# ------------------------------------------------------------------------------------------------ edge cases
@pytest.mark.parametrize('n_fft,hop,n_mels', [(256, 128, 32), (2048, 512, 80)])
def test_melspectrogram_fft_sizes(n_fft, hop, n_mels):
    """All power-of-two FFT sizes of the Stockham kernel (256 = 4^4, 2048 = 4^5 * 2: radix-2 tail pass)."""
    import warnings
    from oracle import frontend as ofe
    margs = dict(sample_rate=16000, n_fft=n_fft, hop_length=hop, n_mels=n_mels)
    g = torch.Generator().manual_seed(n_fft)
    w = torch.randn(2, 20000, generator=g) * 0.1
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')
        ref = ofe.featurize(w, None, 'MelSpectrogram', margs)
        fz = _featurizer(dict(feature_method='MelSpectrogram', method_args=margs))
    got = fz(w).cpu()
    assert got.shape == ref.shape
    assert ((got - ref).abs().max() / ref.abs().max()).item() < 2e-6


def test_short_and_long_utterances(manifest):
    """Shortest accepted audio (min_duration 0.3 s -> 28 frames) and a 14 s utterance (T = 1398 > 800: the attentive
    pooling kernel leaves its shared-memory path; CAM++ gets 7 context segments)."""
    from oracle import frontend as ofe
    from oracle import models as om
    for name in ('ecapa_small', 'campplus_small'):
        m = manifest[name]
        _, sd = load_golden(name)
        model = _model(m['model'], m['feature_dim'], m['model_args'], sd)
        fz = _featurizer(m['preprocess'])
        for lens, seed in (([4800], 1), ([224000, 100000], 2)):
            waves = _ragged(lens, seed)
            x, ratio = ofe.pad_batch(waves)
            fa, fm = m['preprocess']['feature_method'], m['preprocess']['method_args']
            rr = None if len(lens) == 1 else ratio
            ref = om.forward(m['model'], sd, ofe.featurize(x, rr, fa, fm), **m['model_args']).numpy()
            got = model(fz(torch.from_numpy(x), None if rr is None else torch.from_numpy(rr))).cpu().numpy()
            assert rel_l2(got, ref).max() < EMB_TOL, (name, lens)


def test_batch_of_one_and_odd_batches():
    """M tails: B*T not a multiple of the 128-row MMA tile, B = 1 (tiny-M engine selection)."""
    from oracle import models as om
    margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
    sd = om.random_state_dict('EcapaTdnn', 80, seed=11, **margs)
    model = _model('EcapaTdnn', 80, margs, sd)
    g = torch.Generator().manual_seed(4)
    for B, T in ((1, 61), (5, 333), (7, 101)):
        feats = torch.randn(B, T, 80, generator=g) * 2.0
        ref = om.forward('EcapaTdnn', sd, feats, **margs).numpy()
        got = model(feats.cuda()).cpu().numpy()
        assert rel_l2(got, ref).max() < EMB_TOL, (B, T)


def test_extract_features_npy_cache(tmp_path):
    """SURVEY.md 8(f) row 2: MVectorTrainer.extract_features (trainer.py:146-175) writes the [T, F] float32 .npy cache
    + ``*_features.txt`` lists that the reference's reader consumes (reader.py:76-81)."""
    from mvector.trainer import MVectorTrainer
    from oracle import frontend as ofe
    g = torch.Generator().manual_seed(9)
    lists = {}
    for nm, lens in (('train', [16000, 2000, 24000]), ('enroll', [12000]), ('trials', [9000])):
        lines = []
        for i, n in enumerate(lens):
            p = tmp_path / f'{nm}_{i}.wav'
            pcm = (torch.randn(n, generator=g) * 3000).to(torch.int16).numpy()
            with wave.open(str(p), 'wb') as w:
                w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000); w.writeframes(pcm.astype('<i2').tobytes())
            lines.append(f'{p}\t{i}')
        lp = tmp_path / f'{nm}_list.txt'
        lp.write_text('\n'.join(lines) + '\n')
        lists[nm] = str(lp)
    fargs = dict(sample_frequency=16000, num_mel_bins=80)
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'sample_rate': 16000, 'use_dB_normalization': True,
                                        'target_dB': -20},
                            'train_list': lists['train'], 'enroll_list': lists['enroll'], 'trials_list': lists['trials']},
           'preprocess_conf': {'feature_method': 'Fbank', 'method_args': fargs}}
    MVectorTrainer(cfg, use_gpu=True).extract_features(save_dir=str(tmp_path / 'features'), max_duration=1.2)
    out = (tmp_path / 'train_list_features.txt').read_text().splitlines()
    assert len(out) == 3                                 # the 0.125 s file is replaced by its successor (reader.py:86-88)
    for ln in out + (tmp_path / 'enroll_list_features.txt').read_text().splitlines():
        path, label = ln.split('\t')
        f = np.load(path)
        assert f.dtype == np.float32 and f.ndim == 2 and f.shape[1] == 80
        assert f.shape[0] <= 1 + (int(1.2 * 16000) - 400) // 160          # cropped to max_duration
    # content check of the first file against the oracle
    from mvector.audio import AudioSegment
    seg = AudioSegment.from_file(str(tmp_path / 'train_0.wav'))
    seg.normalize(-20)
    ref = ofe.featurize(seg.samples, None, 'Fbank', fargs)[0].numpy()
    got = np.load(out[0].split('\t')[0])
    assert got.shape == ref.shape and np.abs(got - ref).max() < FBANK_ABS_TOL


def test_evaluate_matches_reference_golden(tmp_path, manifest):
    """SURVEY.md 8(f) row 1: MVectorTrainer.evaluate (trainer.py:403-485) on the 3-speaker wav set that the REFERENCE's
    own evaluate was run on (tests/golden/evaluate_small.npz): same eval-order score list (duration sort, singly
    featurized, feature-level zero padding per batch of 4) and the same EER / minDCF / threshold."""
    from mvector.trainer import MVectorTrainer
    import mvector.trainer as mt
    m = manifest['evaluate_small']
    z = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'evaluate_small.npz'))
    lists = {}
    for nm, count in (('enroll', m['n_enroll']), ('trials', m['n_trials'])):
        lines = []
        for i in range(count):
            p = tmp_path / f'{nm}_{i}.wav'
            with wave.open(str(p), 'wb') as w:
                w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000)
                w.writeframes(z[f'{nm}_pcm{i}'].astype('<i2').tobytes())
            lines.append(f'{p}\t{int(z[f"{nm}_label{i}"])}\n')
        lp = tmp_path / f'{nm}_list.txt'
        lp.write_text(''.join(lines))
        lists[nm] = str(lp)
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('sd/')}
    mdir = tmp_path / 'model'
    mdir.mkdir()
    torch.save({'0.' + k: v for k, v in sd.items()}, str(mdir / 'model.pth'))
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': True, 'target_dB': -20},
                            'eval_conf': dict(m['eval_conf']), 'enroll_list': lists['enroll'],
                            'trials_list': lists['trials']},
           'preprocess_conf': {'feature_method': 'Fbank', 'method_args': dict(m['preprocess']['method_args'])},
           'model_conf': {'model': m['model'], 'model_args': dict(m['model_args'])}}
    captured = {}
    real = mt.compute_fnr_fpr

    def spy(scores, labels, weights=None):
        captured['scores'], captured['labels'] = scores.copy(), labels.copy()
        return real(scores, labels, weights)

    mt.compute_fnr_fpr = spy
    try:
        eer, min_dcf, thr = MVectorTrainer(cfg, use_gpu=True).evaluate(resume_model=str(mdir))
    finally:
        mt.compute_fnr_fpr = real
    assert np.array_equal(captured['labels'], z['labels'])
    assert np.abs(captured['scores'] - z['scores']).max() < 2e-5          # cosine scores, embeddings within 1e-4 rel-L2
    assert abs(eer - float(z['eer'])) < 1e-6 and abs(min_dcf - float(z['min_dcf'])) < 1e-6
    assert abs(thr - float(z['threshold'])) < 2e-5


def test_speaker_diarization_flow(manifest):
    """SURVEY.md 8(f) row 4: MVectorPredictor.speaker_diarization (predict.py:365-395) = VAD segments -> 1.5 s chunks ->
    predict_batch on the device -> spectral clustering -> post-processing.  The chunk embeddings are checked against the
    oracle; the host glue is pinned on the reference's own classes by tests/test_host_logic.py."""
    from mvector.predict import MVectorPredictor
    from oracle import frontend as ofe, models as om
    m = manifest['ecapa_small']
    _, sd = load_golden('ecapa_small')
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        pred = MVectorPredictor(configs=_cfg(m['model'], m['model_args'], m['preprocess']), model_path=td, use_gpu=True)
    rng = np.random.RandomState(4)
    t = np.arange(16000 * 4) / 16000.0

    def voice(f0, seed):                   # a "speaker" = harmonic stack + a little noise
        x = sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 9))
        return (0.1 * x + 0.01 * np.random.RandomState(seed).randn(t.size)).astype(np.float32)

    gap = np.zeros(8000, dtype=np.float32)
    x = np.concatenate([gap, voice(110.0, 1), gap, voice(290.0, 2), gap, voice(110.0, 3), gap])
    out = pred.speaker_diarization(x, sample_rate=16000, speaker_num=2)
    assert isinstance(out, list) and len(out) >= 2
    assert all(set(o) == {'speaker', 'start', 'end'} and o['end'] > o['start'] for o in out)
    assert all(a['end'] <= b['start'] + 1e-6 for a, b in zip(out[:-1], out[1:]))
    assert {o['speaker'] for o in out} <= {0, 1} and 0.0 <= out[0]['start'] and out[-1]['end'] <= x.size / 16000.0 + 1e-6
    # the device embeddings of the chunks equal the oracle's on the same padded batch
    from mvector.audio import AudioSegment
    segs = pred.speaker_diarize.segments_audio(AudioSegment(x, 16000))
    chunks = [s[2] for s in segs]
    emb = pred.predict_batch(chunks)
    xb, ratio = ofe.pad_batch(chunks)
    feats = ofe.featurize(xb, ratio, m['preprocess']['feature_method'], m['preprocess']['method_args'])
    ref = om.forward(m['model'], sd, feats, **m['model_args']).numpy()
    assert rel_l2(emb, ref).max() < EMB_TOL


def test_tc_f16_split_runs_and_tf32_fallback_agrees():
    """ENGINE_AUTO routes the wide pointwise / conv layers to conv_tc_kernel<0, true> (kind::f16, hi/lo fp16 terms, dynamic
    activation scale).  Gate: the same 1e-4 embedding parity against the oracle, and the fp16 engine must actually have
    run; with VPB_TC_F16=0 the same models stay on split TF32 and pass the same gate."""
    import subprocess
    import sys
    code = r'''
import sys, numpy as np, torch
sys.path.insert(0, 'tests'); sys.path.insert(0, '.')
from loguru import logger; logger.remove()
from oracle import models as om
from mvector import _lib as L
from mvector.models import build_model
from mvector.utils.utils import dict_to_object
worst = 0.0
for name, fdim, margs, B, T in (('EcapaTdnn', 80, dict(embd_dim=192), 8, 298), ('TDNN', 80, dict(embd_dim=192), 8, 218),
                               ('ResNetSE', 64, dict(embd_dim=192), 2, 151)):
    sd = om.random_state_dict(name, fdim, seed=3, gain=om.CONDITIONED_GAIN[name], **margs)
    m = build_model(fdim, dict_to_object({'model_conf': {'model': name, 'model_args': margs}}))
    m.load_state_dict({'0.' + k: v for k, v in sd.items()})
    x = torch.randn(B, T, fdim, generator=torch.Generator().manual_seed(1)) * 2
    ref = om.forward(name, sd, x, **margs).numpy()
    prog = m.program(B, T)
    emb = torch.empty(B, m.embd_dim, device='cuda')
    ops = prog.run_profiled(x.cuda().contiguous(), emb)
    assert any(o['engine'] == L.ENGINE_TC16 for o in ops), name + ': fp16 engine not selected'
    got = emb.cpu().numpy()
    err = float((np.linalg.norm(got - ref, axis=1) / np.linalg.norm(ref, axis=1)).max())
    print(name, 'rel-L2', err, 'fp16 ops', sum(o['engine'] == L.ENGINE_TC16 for o in ops))
    worst = max(worst, err)
assert worst < 1e-4, worst
print('TC_F16_OK')
'''
    env = dict(os.environ, VPB_TC_F16='1')
    r = subprocess.run([sys.executable, '-c', code], env=env, capture_output=True, text=True, timeout=900,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0 and 'TC_F16_OK' in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    off = code.replace("assert any(o['engine'] == L.ENGINE_TC16 for o in ops), name + ': fp16 engine not selected'",
                       "assert not any(o['engine'] == L.ENGINE_TC16 for o in ops), name + ': fp16 engine ran with VPB_TC_F16=0'")
    r = subprocess.run([sys.executable, '-c', off], env=dict(os.environ, VPB_TC_F16='0'), capture_output=True, text=True,
                       timeout=900, cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert r.returncode == 0 and 'TC_F16_OK' in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_c_host_example_matches_python_host(tmp_path):
    """The same exported program through examples/embed_from_c.c (C, cudart only) and through the Python host."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    from tools import export_program as ex
    from oracle import models as om
    margs = dict(embd_dim=192)
    sd = om.random_state_dict('EcapaTdnn', 80, seed=2, **margs)
    model = _model('EcapaTdnn', 80, margs, sd)
    B, T = 8, 298
    path = str(tmp_path / 'ecapa.vpb')
    ex.export(model, B, T, path)
    feats = (torch.randn(B, T, 80, generator=torch.Generator().manual_seed(4)) * 2).contiguous()
    feats.numpy().tofile(str(tmp_path / 'feats.f32'))
    libdir = os.path.join(root, 'voiceprintrecognition-pytorch_b200')
    exe = str(tmp_path / 'embed_from_c')
    r = subprocess.run(['gcc', '-O1', '-I', os.path.join(root, 'include'), '-I', '/usr/local/cuda/include',
                        os.path.join(root, 'examples', 'embed_from_c.c'), '-o', exe, '-L', libdir, '-lvpb200',
                        '-L', '/usr/local/cuda/lib64', '-lcudart', '-lm', '-Wl,-rpath,' + libdir],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe, path, str(tmp_path / 'feats.f32'), str(tmp_path / 'emb.f32')], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(str(tmp_path / 'emb.f32'), dtype=np.float32).reshape(B, 192)
    ref = model(feats.cuda()).cpu().numpy()
    assert np.array_equal(got, ref)                  # same kernels, same program -> bit identical


@pytest.mark.parametrize('n,m,D', [(1, 1, 192), (7, 33, 192), (100, 257, 512), (3, 5, 36)])
def test_cosine_scores_on_device(n, m, D):
    """vp_cosine_scores (retrieval predict.py:169-183, evaluate trainer.py:454-461, diarization affinity
    speaker_diarization.py:254-257) against sklearn-style normalise-then-matmul in float64."""
    from mvector.engine import Engine
    rng = np.random.default_rng(n * 1000 + m)
    a = rng.standard_normal((n, D)).astype(np.float32) * 3
    b = rng.standard_normal((m, D)).astype(np.float32) * 0.01
    eng = Engine()
    got = eng.cosine_scores(a, b).cpu().numpy()
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    ref = (a64 / np.linalg.norm(a64, axis=1, keepdims=True)) @ (b64 / np.linalg.norm(b64, axis=1, keepdims=True)).T
    assert got.shape == (n, m) and np.abs(got - ref).max() < 2e-6
    assert torch.equal(eng.cosine_scores(a, b), eng.cosine_scores(a, b))          # deterministic
    eng.close()
