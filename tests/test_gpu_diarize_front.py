"""Device diarization front (csrc/segment.cu through Engine.frame_energy / gather_windows and
MVectorPredictor.speaker_diarization) against the host flow it replaces: numpy's frame energies, host slicing of the
chunks, and predict_batch on host-built chunks of the device-conditioned recording."""
import os
import tempfile

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MARGS = dict(embd_dim=192, pooling_type='ASP', channels=[128, 128, 128, 128, 384], attention_channels=64,
             res2net_scale=4, se_channels=32)


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    return Engine(0)


def _host_energy(x, hop):
    nf = x.size // hop
    return (x[:nf * hop].astype(np.float64).reshape(nf, hop) ** 2).mean(axis=1)


@pytest.mark.parametrize('hop', [1, 3, 7, 8, 9, 100, 128, 129, 441, 480, 1323, 1440, 2000])
def test_frame_energy_bit_exact(eng, hop):
    rng = np.random.default_rng(hop)
    for n in (hop - 1, hop, 37 * hop + hop // 3, 1000 * hop + 1):
        if n < 0:
            continue
        x = (rng.standard_normal(n) * rng.uniform(1e-4, 4)).astype(np.float32)
        got = eng.frame_energy(torch.from_numpy(x).cuda(), n, hop).cpu().numpy()
        ref = _host_energy(x, hop)
        assert got.shape == ref.shape and np.array_equal(got.view(np.uint64), ref.view(np.uint64)), (hop, n)


def test_frame_energy_nan_inf_and_long_row(eng):
    hop = 480
    x = (np.random.default_rng(1).standard_normal(hop * 50) * 0.1).astype(np.float32)
    x[hop * 3 + 17] = np.nan
    x[hop * 9 + 400] = np.inf
    got = eng.frame_energy(torch.from_numpy(x).cuda(), x.size, hop).cpu().numpy()
    ref = _host_energy(x, hop)
    assert np.isnan(got[3]) and np.isinf(got[9])
    ok = np.isfinite(ref)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[~np.isnan(ref)], ref[~np.isnan(ref)])
    assert ok.sum() == 48
    # 2^27 samples (over an hour at 16 kHz) with a hop that does not divide it: the last frames and the int64 row offsets
    n = (1 << 27) + 1234
    g = torch.Generator(device='cuda').manual_seed(2)
    xd = torch.randn(n, generator=g, device='cuda') * 0.3
    got = eng.frame_energy(xd, n, 441).cpu().numpy()
    ref = _host_energy(xd.cpu().numpy(), 441)
    assert got.shape == ref.shape and np.array_equal(got.view(np.uint64), ref.view(np.uint64))


def _gather_ref(src, offset, valid, ld):
    out = np.zeros((len(offset), ld), dtype=np.float32)
    for i, (o, v) in enumerate(zip(offset, valid)):
        v = max(0, min(int(v), ld))
        out[i, :v] = src[o:o + v]
    return out


def test_gather_windows_exact(eng):
    rng = np.random.default_rng(3)
    src = rng.standard_normal(100003).astype(np.float32)
    ld = 24000
    offset = np.array([0, 5, 1000, 100003 - ld, 100003 - 7, 76003, 99, 50000], dtype=np.int64)
    valid = np.array([ld, 0, 123, ld, 7, ld, 1, ld - 1], dtype=np.int32)        # full / empty / partial, ends at the end
    dst = torch.full((len(offset), ld), float('nan'), device='cuda')
    eng.gather_windows(torch.from_numpy(src).cuda(), torch.from_numpy(offset).cuda(), torch.from_numpy(valid).cuda(), ld,
                       dst)
    assert np.array_equal(dst.cpu().numpy(), _gather_ref(src, offset, valid, ld))
    # an odd leading dimension and more rows than one grid column holds
    ld2, rows = 1001, 70000
    off2 = rng.integers(0, src.size - ld2, rows).astype(np.int64)
    val2 = rng.integers(0, ld2 + 1, rows).astype(np.int32)
    dst2 = torch.empty(rows * ld2, device='cuda')
    eng.gather_windows(torch.from_numpy(src).cuda(), torch.from_numpy(off2).cuda(), torch.from_numpy(val2).cuda(), ld2,
                       dst2)
    assert np.array_equal(dst2.view(rows, ld2).cpu().numpy(), _gather_ref(src, off2, val2, ld2))


def test_gather_windows_offset_past_2g_bytes(eng):
    n = (1 << 29) + (1 << 16)                                    # 2 GiB + 256 KiB of float32
    src = torch.arange(n, device='cuda', dtype=torch.int32).to(torch.float32)
    offset = np.array([(1 << 29) + 5, n - 24000, 3], dtype=np.int64)      # byte offsets past 2^31
    valid = np.array([24000, 24000, 100], dtype=np.int32)
    dst = torch.empty(3, 24000, device='cuda')
    eng.gather_windows(src, torch.from_numpy(offset).cuda(), torch.from_numpy(valid).cuda(), 24000, dst)
    want = np.zeros((3, 24000), dtype=np.float32)
    for i, (o, v) in enumerate(zip(offset, valid)):
        want[i, :v] = np.arange(o, o + v).astype(np.float32)
    assert np.array_equal(dst.cpu().numpy(), want)


# ------------------------------------------------------------------------------------------------ predictor
def _predictor(feature, db, td, min_duration=0.3):
    from mvector.predict import MVectorPredictor
    from oracle import models as om
    fargs = dict(sample_frequency=16000, num_mel_bins=80) if feature == 'Fbank' else {}
    dim = 80 if feature == 'Fbank' else 40
    sd = om.random_state_dict('EcapaTdnn', dim, seed=5, **MARGS)
    cfg = {'dataset_conf': {'dataset': {'min_duration': min_duration, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': db, 'target_dB': -20},
                            'eval_conf': {'batch_size': 16, 'max_duration': 20}},
           'preprocess_conf': {'use_hf_model': False, 'feature_method': feature, 'method_args': fargs},
           'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(MARGS)}}
    path = os.path.join(td, f'{feature}.pth')
    torch.save({'0.' + k: v for k, v in sd.items()}, path)
    return MVectorPredictor(configs=cfg, model_path=path, use_gpu=True)


@pytest.fixture(scope='module')
def preds():
    with tempfile.TemporaryDirectory() as td:
        return {'on': _predictor('Fbank', True, td), 'off': _predictor('Fbank', False, td),
                'mfcc': _predictor('MFCC', True, td)}


def _recording(sr, seconds=24.0, seed=0):
    """Two synthetic speakers taking turns, with pauses, at ``sr`` Hz."""
    rng = np.random.RandomState(seed)
    parts = []
    for k in range(int(seconds // 4)):
        d = rng.uniform(2.0, 3.4)
        t = np.arange(int(d * sr)) / float(sr)
        f0 = (110.0, 290.0)[k % 2] * rng.uniform(0.97, 1.03)
        v = sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 9))
        parts.append((0.1 * v + 0.01 * rng.randn(t.size)).astype(np.float32))
        parts.append(np.zeros(int(rng.uniform(0.4, 0.9) * sr), dtype=np.float32))
    return np.concatenate(parts)


def _conditioned(pred, x, sr):
    """The recording as speaker_diarization conditions it: on the device (Engine.condition)."""
    ds = pred.configs.dataset_conf.dataset
    y, n_out, _ = pred._engine.condition(torch.from_numpy(x).cuda().view(1, -1), [x.size], [sr], 16000,
                                         ds.target_dB if ds.use_dB_normalization else None)
    return y[0, :int(n_out[0])].cpu().numpy()


def _host_construction(pred, y16, sample_rate, speaker_num, search=False):
    """The host flow on the device-conditioned recording: segments_audio -> predict_batch -> clustering -> postprocess."""
    from mvector.audio import AudioSegment
    segments = pred.speaker_diarize.segments_audio(AudioSegment(y16.copy(), 16000))
    feats = pred.predict_batch([s[2] for s in segments], sample_rate=sample_rate)
    np.random.seed(0)
    labels, centres = pred.speaker_diarize.clustering(feats, speaker_num=speaker_num)
    out = pred.speaker_diarize.postprocess(segments, labels)
    if search:
        names = pred._MVectorPredictor__retrieval(np_feature=centres)
        out = [{'speaker': names[o['speaker']][0] if names[o['speaker']][0] else f"陌生人{o['speaker']}",
                'start': o['start'], 'end': o['end']} for o in out]
    return feats, out


def _device(pred, audio, sample_rate, speaker_num, search=False):
    captured = {}
    real = pred.speaker_diarize.clustering

    def clustering(features, speaker_num=None):
        captured['feats'] = np.array(features, copy=True)
        np.random.seed(0)
        return real(features, speaker_num=speaker_num)
    pred.speaker_diarize.clustering = clustering
    try:
        out = pred.speaker_diarization(audio, sample_rate=sample_rate, speaker_num=speaker_num, search_audio_db=search)
    finally:
        del pred.speaker_diarize.clustering
    return captured['feats'], out


CASES = [  # (predictor, native rate, caller sample_rate or None for the native one, speaker_num)
    ('on', 16000, None, None),
    ('on', 8000, None, 2),
    ('on', 44100, None, None),
    ('on', 48000, None, 2),
    ('off', 48000, None, None),
    ('off', 16000, None, 2),
    ('on', 44100, 16000, 2),          # a file-like input at 44.1 kHz, the caller's default rate for the chunks
    ('on', 16000, 48000, None),       # chunks passed on as 48 kHz: resampled a second time
    ('off', 8000, 22050, 2),
    ('mfcc', 16000, None, 2),
    ('mfcc', 44100, 16000, None),
]


@pytest.mark.parametrize('key,native,caller,k', CASES)
def test_speaker_diarization_equals_host_construction(preds, key, native, caller, k):
    from mvector.audio import AudioSegment
    pred = preds[key]
    x = _recording(native, seed=native % 97)
    y16 = _conditioned(pred, x, native)
    if caller is None:
        feats, out = _device(pred, x, native, k)
        rate = native
    else:
        feats, out = _device(pred, AudioSegment(x.copy(), native), caller, k)
        rate = caller
    ref_feats, ref_out = _host_construction(pred, y16, rate, k)
    assert feats.shape == ref_feats.shape and np.array_equal(feats, ref_feats)
    assert out == ref_out and len(out) >= 2


def test_device_conditioned_recording_within_one_ulp_of_host(preds):
    from mvector.audio import AudioSegment
    for key in ('on', 'off'):
        pred = preds[key]
        for sr in (8000, 16000, 44100, 48000):
            x = _recording(sr, seed=sr % 89)
            host = pred._condition_host(AudioSegment(x.copy(), sr)).samples
            dev = _conditioned(pred, x, sr)
            assert dev.shape == host.shape
            u = np.abs(dev.view(np.int32).astype(np.int64) - host.view(np.int32).astype(np.int64))
            assert u.max() <= (1 if key == 'on' else 0), (key, sr, int(u.max()))


def test_search_audio_db(preds):
    pred = preds['on']
    x = _recording(16000, seed=4)
    y16 = _conditioned(pred, x, 16000)
    rng = np.random.RandomState(5)
    ref_feats, _ = _host_construction(pred, y16, 16000, 2)
    pred.audio_feature = ref_feats[:2].copy()
    pred.audio_feature_mean = np.stack([ref_feats[0], rng.randn(ref_feats.shape[1]).astype(np.float32)])
    pred.users_name_mean = ['alice', 'bob']
    pred.threshold = -1.0                    # every speaker gets the closer of the two names
    try:
        _, want = _host_construction(pred, y16, 16000, 2, search=True)
        _, got = _device(pred, x, 16000, 2, search=True)
    finally:
        pred.audio_feature = pred.audio_feature_mean = None
        pred.users_name_mean = []
        pred.threshold = 0.6
    assert got == want and any(o['speaker'] == 'alice' for o in got)


def _raised(fn):
    try:
        fn()
    except (AssertionError, ValueError) as e:
        return type(e), str(e)
    return None


def test_error_paths_raise_what_the_host_flow_raises(preds, monkeypatch):
    from mvector.audio import AudioSegment
    pred = preds['on']

    def host_flow(audio, sample_rate):
        seg = pred._condition_host(pred._load_audio(audio, sample_rate))
        segments = pred.speaker_diarize.segments_audio(seg)
        pred.predict_batch([s[2] for s in segments], sample_rate=sample_rate)

    def both(make, sample_rate):              # make(): a fresh input (_condition_host works in place)
        a = _raised(lambda: host_flow(make(), sample_rate))
        b = _raised(lambda: pred.speaker_diarization(make(), sample_rate=sample_rate))
        assert a is not None and a == b, (a, b)
        return a[0]
    # the recording's own too-short assert, at its native duration
    assert both(lambda: np.ones(int(48000 * 0.3) - 3, dtype=np.float32), 48000) is AssertionError
    # a silent recording cannot be normalised
    assert both(lambda: np.zeros(16000 * 8, dtype=np.float32), 16000) is ValueError
    # < 5 s of speech
    assert both(lambda: _recording(16000, seconds=8.0)[:16000 * 4], 16000) is AssertionError
    # chunks of 24000 samples passed on as 96 kHz are 0.25 s: predict_batch's too-short assert
    assert both(lambda: AudioSegment(_recording(16000), 16000), 96000) is AssertionError
    # a silent chunk: the VAD made to keep a long pause
    x = np.concatenate([_recording(16000, seconds=8.0, seed=2), np.zeros(16000 * 3, dtype=np.float32),
                        _recording(16000, seconds=8.0, seed=3)])

    def keep_all(ms, n, sr, return_seconds=False, *args, **kw):
        return [{'start': 0.0, 'end': n / sr} if return_seconds else {'start': 0, 'end': n}]
    monkeypatch.setattr(AudioSegment, 'vad_from_energy', staticmethod(keep_all))
    assert both(lambda: x.copy(), 16000) is ValueError


def test_speaker_diarization_keeps_the_recording_on_the_device(preds, monkeypatch):
    from mvector import _lib as L
    from mvector.audio import AudioSegment
    from mvector.predict import MVectorPredictor
    pred = preds['on']
    calls = []
    lib = L.lib()
    real = lib.vp_host_stage_h2d
    monkeypatch.setattr(lib, 'vp_host_stage_h2d', lambda *a: calls.append('vp_host_stage_h2d') or real(*a))
    monkeypatch.setattr(AudioSegment, 'vad', lambda *a, **k: calls.append('vad') or [])
    monkeypatch.setattr(MVectorPredictor, '_condition_host', lambda *a, **k: calls.append('_condition_host'))
    out = pred.speaker_diarization(_recording(44100, seed=8), sample_rate=44100, speaker_num=2)
    assert calls == [] and len(out) >= 2
