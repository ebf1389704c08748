"""Device input conditioning (csrc/condition.cu through Engine.condition and the predictor's staging) against the host
conditioning it replaces: AudioSegment.resample (scipy's resample_poly) and AudioSegment.normalize."""
import os
import socket
import tempfile
import wave

import numpy as np
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu

RATES = (8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000, 96000)
MARGS = dict(embd_dim=192, pooling_type='ASP', channels=[128, 128, 128, 128, 384], attention_channels=64,
             res2net_scale=4, se_channels=32)
FARGS = dict(sample_frequency=16000, num_mel_bins=80)


def _host(x, sr, db=True):
    from mvector.audio import AudioSegment
    seg = AudioSegment(np.array(x, dtype=np.float32, copy=True), sr)
    seg.resample(16000)
    if db:
        seg.normalize(target_db=-20)
    return seg.samples


def _ulps(a, b):
    ia = np.asarray(a, dtype=np.float32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, dtype=np.float32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    return Engine(0)


def _batch(seed, rates, lens):
    rng = np.random.default_rng(seed)
    waves = [(rng.standard_normal(n) * rng.uniform(0.01, 0.5)).astype(np.float32) for n in lens]
    ld = max(lens)
    x = np.zeros((len(lens), ld), dtype=np.float32)
    for i, w in enumerate(waves):
        x[i, :len(w)] = w
    return waves, torch.from_numpy(x).cuda()


def test_mixed_rate_batch_resample_is_bit_identical(eng):
    rng = np.random.default_rng(0)
    rates = list(RATES) + [16000] + list(RATES)
    lens = [1, 17, 250] + [int(rng.integers(r // 3, 2 * r)) for r in rates[3:]]
    waves, x = _batch(1, rates, lens)
    y, n_out, flags = eng.condition(x, lens, rates, 16000)
    assert flags is None
    y = y.cpu().numpy()
    for i, (w, r) in enumerate(zip(waves, rates)):
        ref = _host(w, r, db=False)
        assert n_out[i] == ref.size
        assert np.array_equal(y[i, :ref.size], ref), (r, lens[i])
        assert not y[i, ref.size:].any()                     # padding exactly zero
    y2, _, _ = eng.condition(x, lens, rates, 16000)
    assert np.array_equal(y2.cpu().numpy(), y)               # two runs bit-identical


def test_normalised_rows_within_the_factor_contract(eng):
    rng = np.random.default_rng(2)
    rates = [RATES[i % len(RATES)] for i in range(40)] + [16000] * 8
    lens = [int(rng.integers(r // 2, 3 * r)) for r in rates]
    waves, x = _batch(3, rates, lens)
    y, n_out, flags = eng.condition(x, lens, rates, 16000, target_db=-20)
    y = y.cpu().numpy()
    assert not flags.cpu().numpy().any()
    differ = 0
    for i, (w, r) in enumerate(zip(waves, rates)):
        ref = _host(w, r)
        u = _ulps(y[i, :ref.size], ref)
        assert u.max() <= 1, (r, int(u.max()))
        differ += int(u.any())
        assert not y[i, ref.size:].any()
    print(f'rows whose normalised samples differ from AudioSegment.normalize (1 ulp allowed): {differ} of {len(rates)}')
    y2, _, _ = eng.condition(x, lens, rates, 16000, target_db=-20)
    assert np.array_equal(y2.cpu().numpy(), y)


def test_nan_propagates_and_silence_is_flagged(eng):
    lens = [48000, 48000, 32000]
    rates = [48000, 16000, 16000]
    waves, x = _batch(4, rates, lens)
    x[0, 100] = float('nan')
    x[2] = 0
    y, n_out, flags = eng.condition(x, lens, rates, 16000, target_db=-20)
    y, fl = y.cpu().numpy(), flags.cpu().numpy()
    assert fl.tolist() == [0, 0, 1]
    assert np.isnan(y[0, :n_out[0]]).all()                   # the host's mean is NaN too: the whole row
    ref = _host(waves[1], 16000)
    assert _ulps(y[1, :ref.size], ref).max() <= 1
    with pytest.raises(ValueError):
        _host(np.zeros(32000, dtype=np.float32), 16000)


# ------------------------------------------------------------------------------------------------ predictor
def _predictor(sd, db, td):
    from mvector.predict import MVectorPredictor
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': db, 'target_dB': -20},
                            'eval_conf': {'batch_size': 16, 'max_duration': 20}},
           'preprocess_conf': {'use_hf_model': False, 'feature_method': 'Fbank', 'method_args': dict(FARGS)},
           'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(MARGS)}}
    torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
    return MVectorPredictor(configs=cfg, model_path=td, use_gpu=True)


@pytest.fixture(scope='module')
def preds():
    from oracle import models as om
    sd = om.random_state_dict('EcapaTdnn', 80, seed=5, **MARGS)
    with tempfile.TemporaryDirectory() as td:
        return _predictor(sd, True, td), _predictor(sd, False, td)


def _wav(path, x, sr):
    pcm = (np.clip(x, -1, 1) * 32767).astype('<i2')
    with wave.open(str(path), 'wb') as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(sr); w.writeframes(pcm.tobytes())
    return str(path)


def test_predictor_normalise_on_equals_host_conditioned(preds, tmp_path):
    from mvector.audio import AudioSegment
    pn, pp = preds
    rng = np.random.default_rng(6)
    x48 = [(rng.standard_normal(int(rng.integers(20000, 150000))) * 0.2).astype(np.float32) for _ in range(5)]
    assert np.array_equal(pn.predict_batch(x48, sample_rate=48000),
                          pp.predict_batch([_host(x, 48000) for x in x48]))
    files, host = [], []
    for i, sr in enumerate((8000, 16000, 44100, 8000, 44100)):
        x = (rng.standard_normal(int(sr * rng.uniform(0.5, 2.5))) * 0.3).astype(np.float32)
        p = _wav(tmp_path / f'{i}.wav', x, sr)
        files.append(p)
        seg = AudioSegment.from_file(p)
        host.append(_host(seg.samples, seg.sample_rate))
    assert np.array_equal(pn.predict_batch(files), pp.predict_batch(host))
    segs = [AudioSegment.from_file(p) for p in files]
    assert np.array_equal(pn.predict_batch(segs), pp.predict_batch(host))
    assert np.array_equal(pn.predict(files[2]), pp.predict(host[2]))
    assert np.array_equal(pn.predict(x48[0], sample_rate=48000), pp.predict(_host(x48[0], 48000)))
    assert pn.contrast(files[0], files[2]) == pp.contrast(host[0], host[2])
    with pytest.raises(AssertionError):                     # the too-short assert is on the NATIVE duration
        pn.predict(np.ones(48000 * 3 // 10 - 3, dtype=np.float32), sample_rate=48000)
    with pytest.raises(ValueError):                          # a silent item cannot be normalised
        pn.predict_batch([x48[1], np.zeros(16000, dtype=np.float32)])


def test_speaker_diarization_48k_equals_host_construction(preds):
    from mvector.audio import AudioSegment
    pn, pp = preds
    t = np.arange(48000 * 4) / 48000.0

    def voice(f0, seed):
        v = sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 9))
        return (0.1 * v + 0.01 * np.random.RandomState(seed).randn(t.size)).astype(np.float32)

    gap = np.zeros(24000, dtype=np.float32)
    x = np.concatenate([gap, voice(110.0, 1), gap, voice(290.0, 2), gap, voice(110.0, 3), gap])
    got = pn.speaker_diarization(x, sample_rate=48000, speaker_num=2)
    seg = AudioSegment(x.copy(), 48000)
    seg.resample(16000)
    seg.normalize(target_db=-20)
    segments = pp.speaker_diarize.segments_audio(seg)
    # the reference passes the 16 kHz chunks on with the caller's rate: they are resampled a second time
    feats = pp.predict_batch([_host(s[2], 48000) for s in segments])
    labels, _ = pp.speaker_diarize.clustering(feats, speaker_num=2)
    assert got == pp.speaker_diarize.postprocess(segments, labels)


def test_plain_16k_call_enqueues_no_conditioning(preds, monkeypatch):
    from mvector import _lib as L
    pn, pp = preds
    lib = L.lib()
    calls = []
    for name in ('vp_resample', 'vp_gain_normalize'):
        real = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *a, _n=name, _r=real: calls.append(_n) or _r(*a))
    x = [np.random.default_rng(8).standard_normal(32000).astype(np.float32) * 0.1 for _ in range(3)]
    pp.predict_batch(x)
    assert calls == []
    pn.predict_batch(x, sample_rate=48000)
    assert 'vp_resample' in calls and 'vp_gain_normalize' in calls


def test_trainer_features_and_evaluate_at_44k(tmp_path):
    from mvector.trainer import MVectorTrainer
    from mvector.audio import AudioSegment
    from oracle import models as om
    rng = np.random.default_rng(11)
    lines = []
    for i in range(6):
        p = _wav(tmp_path / f'a{i}.wav', (rng.standard_normal(int(44100 * (1 + i * 0.4))) * 0.2).astype(np.float32), 44100)
        lines.append(f'{p}\t{i % 3}\n')
    (tmp_path / 'list.txt').write_text(''.join(lines))
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': True, 'target_dB': -20},
                            'eval_conf': {'batch_size': 4, 'max_duration': 2}, 'train_list': str(tmp_path / 'list.txt'),
                            'enroll_list': str(tmp_path / 'list.txt'), 'trials_list': str(tmp_path / 'list.txt')},
           'preprocess_conf': {'feature_method': 'Fbank', 'method_args': dict(FARGS)},
           'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(MARGS)}}
    tr = MVectorTrainer(cfg, use_gpu=True)
    tr._setup_eval()
    sd = om.random_state_dict('EcapaTdnn', 80, seed=5, **MARGS)
    tr.model.load_state_dict(sd)
    for ln in lines:
        path = ln.split('\t')[0]
        got = tr._eval_feature(path).cpu().numpy()
        seg = AudioSegment.from_file(path)
        host = _host(seg.samples, seg.sample_rate)[:int(2 * 16000)]
        ref = tr.audio_featurizer(torch.from_numpy(host)).squeeze(0).cpu().numpy()
        assert np.array_equal(got, ref)
    eer, min_dcf, thr = tr.evaluate()
    assert 0.0 <= eer <= 1.0 and np.isfinite(min_dcf)
    tr.extract_features(save_dir=str(tmp_path / 'features'), max_duration=1.5)
    out = (tmp_path / 'list_features.txt').read_text().splitlines()
    seg = AudioSegment.from_file(lines[2].split('\t')[0])
    host = _host(seg.samples, seg.sample_rate)[:int(1.5 * 16000)]
    ref = tr.audio_featurizer(torch.from_numpy(host)).squeeze(0).cpu().numpy()
    assert np.array_equal(np.load(out[2].split('\t')[0]), ref)


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, out_dir):
    import sys
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(0)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, 'tests')):
        if p not in sys.path:
            sys.path.insert(0, p)
    from mvector.distributed import predict_batch_sharded
    from oracle import models as om
    sd = om.random_state_dict('EcapaTdnn', 80, seed=5, **MARGS)
    with tempfile.TemporaryDirectory() as td:
        pred = _predictor(sd, True, td)
    rng = np.random.default_rng(12)
    waves = [(rng.standard_normal(n) * a).astype(np.float32)
             for n, a in zip([44100, 132300, 30001, 90000, 15000, 60000, 200000], [0.1, 0.3, 0.05, 0.2, 1e-3, 0.1, 0.1])]
    full = pred.predict_batch(waves, sample_rate=44100)
    got = predict_batch_sharded(pred, waves, sample_rate=44100)
    np.save(os.path.join(out_dir, f'rank{rank}.npy'), np.stack([full, got]))
    dist.barrier()
    dist.destroy_process_group()


def test_predict_batch_sharded_44k_normalised_two_ranks_one_gpu():
    """Split-TF32 engine (VPB_TC_F16=0): bit exact; default FP16 split: <= 2e-6 relative L2 (the activation scale of a
    layer follows the tensor the kernel sees -- the whole batch or the shard)."""
    import torch.multiprocessing as mp
    for f16, tol in (('0', 0.0), ('1', 2e-6)):
        old = os.environ.get('VPB_TC_F16')
        os.environ['VPB_TC_F16'] = f16
        try:
            with tempfile.TemporaryDirectory() as td:
                mp.spawn(_sharded_worker, args=(2, _free_port(), td), nprocs=2, join=True)
                for r in range(2):
                    full, got = np.load(os.path.join(td, f'rank{r}.npy'))
                    if tol == 0.0:
                        assert np.array_equal(full, got), (r, np.abs(full - got).max())
                    else:
                        assert rel_l2(got, full).max() <= tol
        finally:
            if old is None:
                os.environ.pop('VPB_TC_F16', None)
            else:
                os.environ['VPB_TC_F16'] = old
