"""Device conversion of uncompressed PCM containers (csrc/pcm.cu through Engine.decode_pcm) against the host
conversion (PcmSegment.samples, itself checked against pcm_oracle.py by test_pcm_cpu.py), and the callers that read
such files: predict, predict_batch, contrast, speaker_diarization, evaluate and extract_features give what the same
samples give as float32 arrays, or as 16-bit WAV where that is exact."""
import dataclasses
import io
import os
import tempfile
import wave

import numpy as np
import pytest

import flac_writer as fw
import pcm_oracle as po
import pcm_writer as pw

pytestmark = pytest.mark.gpu

MARGS = dict(embd_dim=192, pooling_type='ASP', channels=[128, 128, 128, 128, 384], attention_channels=64,
             res2net_scale=4, se_channels=32)
FARGS = dict(sample_frequency=16000, num_mel_bins=80)


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    return Engine(0)


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


def _host(data):
    from mvector.audio import AudioSegment
    return AudioSegment.from_bytes(data).samples


def _matrix():
    """The format matrix, then a 24-bit row whose last sample ends on the last byte of the batch."""
    cases = [(name, data) for name, data, *_ in pw.matrix(np.random.default_rng(7))]
    vals = pw.random_samples(np.random.default_rng(8), 's24le', 3 * 41)
    cases.append(('last-s24le-3ch', pw.wav(pw.encode(vals, 's24le'), 44100, 3, 's24le')))
    return cases


def test_matrix_bit_identical_to_host(eng):
    from mvector.pcm import parse_header
    cases = _matrix()
    files = [d for _, d in cases]
    infos = [parse_header(d) for d in files]
    base = np.concatenate([[0], np.cumsum([len(d) for d in files])])[:-1]
    starts = base + np.array([i.data_offset for i in infos])
    assert (starts % 2 == 1).any() and (starts % 4 == 3).any()                     # unaligned rows
    last = infos[-1]
    assert last.data_offset + last.frames * 3 * 3 == len(files[-1])               # ends on the batch's last byte
    ld = max(i.frames for i in infos) + 37
    rows, status = eng.decode_pcm(files, names=[n for n, _ in cases], ld=ld)
    rows, status = rows.cpu().numpy(), status.cpu().numpy()
    assert not status.any()
    for i, (name, data) in enumerate(cases):
        ref = _host(data)
        assert np.array_equal(_bits(rows[i, :ref.size]), _bits(ref)), name
        assert not rows[i, ref.size:].any(), name                                 # zero fill to ld
    again, _ = eng.decode_pcm(files, infos, ld=ld)
    assert np.array_equal(_bits(again.cpu().numpy()), _bits(rows))


def test_refused_rows_leave_the_others_exact(eng):
    from mvector.pcm import parse_header
    vals = pw.random_samples(np.random.default_rng(9), 's16be', 2 * 300)
    good = pw.aiff(pw.encode(vals, 's16be'), 16000, 2, 300, 's16be')
    gi = parse_header(good)
    ld = gi.frames
    bad = [(dataclasses.replace(gi, format=99), 1), (dataclasses.replace(gi, format=0), 1),
           (dataclasses.replace(gi, channels=0), 2), (dataclasses.replace(gi, channels=9), 2),
           (dataclasses.replace(gi, frames=ld + 1), 4), (dataclasses.replace(gi, frames=-1), 4),
           (dataclasses.replace(gi, data_offset=10 ** 12), 8), (dataclasses.replace(gi, data_offset=-10 ** 6), 8)]
    # row 9 of 11 starts at byte 9 * len(good): its first sample is the batch's last byte, its frames run past it
    bad.append((dataclasses.replace(gi, data_offset=2 * len(good) - 1), 8))
    infos = [gi] + [b for b, _ in bad] + [gi]
    assert len(infos) == 11
    names = ['good-a'] + [f'bad-{k}' for k in range(len(bad))] + ['good-b']
    rows, status = eng.decode_pcm([good] * len(infos), infos, names, ld=ld, check=False)
    st, r = status.cpu().numpy(), rows.cpu().numpy()
    assert list(st) == [0] + [s for _, s in bad] + [0]
    ref = _host(good)
    assert np.array_equal(_bits(r[0]), _bits(ref)) and np.array_equal(_bits(r[-1]), _bits(ref))
    assert not r[1:-1].any()                                                      # refused rows are zeros
    with pytest.raises(ValueError, match='bad-0'):
        eng.decode_pcm([good] * len(infos), infos, names, ld=ld)


def test_empty_rows_and_no_columns(eng):
    """Files of 0 frames: a [B, 0] result and status 0 for every row, not an argument error."""
    empty = [pw.wav(b'', 16000, 1, 's16le'), pw.aiff(b'', 8000, 2, 0, 's24be')]
    rows, status = eng.decode_pcm(empty)
    assert tuple(rows.shape) == (2, 0) and not status.cpu().numpy().any()
    rows, _ = eng.decode_pcm(empty, ld=5)
    assert tuple(rows.shape) == (2, 5) and not rows.cpu().numpy().any()


def test_row_of_2_27_samples(eng):
    import torch
    n = 1 << 27
    x = (np.arange(n, dtype=np.int64) * 7919 % 65536 - 32768).astype('<i2')
    data = pw.wav(x.tobytes(), 16000, 1, 's16le')
    rows, _ = eng.decode_pcm([data])
    assert rows.shape == (1, n)
    expect = torch.from_numpy(x.astype(np.float32) / np.float32(32768)).to(rows.device)
    assert torch.equal(rows[0], expect)


# ------------------------------------------------------------------------------------------------ callers
@pytest.fixture(scope='module')
def preds():
    import torch
    from mvector.predict import MVectorPredictor
    from oracle import models as om
    sd = om.random_state_dict('EcapaTdnn', 80, seed=5, **MARGS)
    out = []
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        for db in (True, False):
            cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                                'use_dB_normalization': db, 'target_dB': -20},
                                    'eval_conf': {'batch_size': 16, 'max_duration': 20}},
                   'preprocess_conf': {'use_hf_model': False, 'feature_method': 'Fbank', 'method_args': dict(FARGS)},
                   'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(MARGS)}}
            out.append(MVectorPredictor(configs=cfg, model_path=td, use_gpu=True))
    return out


def _speech_like(rng, n, ch):
    t = np.arange(n)[:, None]
    x = 6000 * np.sin(2 * np.pi * t * rng.uniform(0.001, 0.05, size=(1, ch))) + rng.normal(0, 800, size=(n, ch))
    return np.clip(np.round(x), -32768, 32767).astype(np.int64)


_MU = np.array([po.ulaw_to_int(b) for b in range(256)])


def _file(ints, rate, kind):
    """int16-range samples [n, ch] as a file of ``kind`` -> (bytes, the float32 mono row the file holds)."""
    n, ch = ints.shape
    flat = ints.reshape(-1)
    fmt, vals, mk = {
        's24le': ('s24le', flat << 8, 'wav'), 'f32le': ('f32le', flat / 32768.0, 'wav'),
        'f64be': ('f64be', flat / 32768.0 + 1e-9, 'aiff'), 'ulaw': ('ulaw', None, 'wav'),
        's16be': ('s16be', flat, 'aiff'), 'alaw': ('alaw', flat & 0xFF, 'aiff'), 'u8': ('u8', (flat >> 8) + 128, 'wav'),
        's16le': ('s16le', flat, 'wav')}[kind]
    if kind == 'ulaw':                                   # a mu-law code at or above every sample
        order = np.argsort(_MU)
        idx = np.clip(np.searchsorted(_MU[order], flat), 0, 255)
        vals = order[idx]
    raw = pw.encode(vals, fmt)
    data = pw.wav(raw, rate, ch, fmt) if mk == 'wav' else pw.aiff(raw, rate, ch, n, fmt)
    return data, po.decode(raw, fmt, ch)


KINDS = ('s24le', 'f32le', 'f64be', 'ulaw', 's16be', 'alaw', 'u8', 's16le')


@pytest.mark.parametrize('db', [0, 1])
def test_predict_from_pcm_files_equals_arrays(preds, db, tmp_path):
    from mvector.audio import AudioSegment
    p = preds[db]
    rng = np.random.default_rng(11 + db)
    items, arrays, rates, paths = [], [], [], []
    for i, rate in enumerate([8000, 16000, 44100, 48000] * 3):
        n = int(rng.integers(int(0.4 * rate), int(1.6 * rate)))
        data, arr = _file(_speech_like(rng, n, 1 + i % 3), rate, KINDS[i % len(KINDS)])
        path = tmp_path / f'{i}.{"aif" if data[:4] == b"FORM" else "wav"}'
        path.write_bytes(data)
        kind = i % 3
        items.append(str(path) if kind == 0 else data if kind == 1 else open(path, 'rb'))
        paths.append(str(path))
        arrays.append(arr)
        rates.append(rate)
    got = p.predict_batch(items)
    ref = p.predict_batch([AudioSegment(a, r) for a, r in zip(arrays, rates)])
    assert np.array_equal(got, ref)
    for k in (0, 3, 5, 7):
        assert np.array_equal(p.predict(paths[k]), p.predict(arrays[k], sample_rate=rates[k]))
        assert np.array_equal(p.predict(io.BufferedReader(io.FileIO(paths[k]))),
                              p.predict(arrays[k], sample_rate=rates[k]))
    c = p.contrast(paths[1], paths[2])
    f1, f2 = p.predict(arrays[1], sample_rate=rates[1]), p.predict(arrays[2], sample_rate=rates[2])
    assert c == np.dot(f1, f2) / (np.linalg.norm(f1) * np.linalg.norm(f2))


def test_pcm_only_call_converts_into_the_staging_slots(preds, tmp_path, monkeypatch):
    """A call whose items are all PCM files never stages host samples (vp_host_stage_h2d) and never reads
    PcmSegment.samples; its embeddings are those of the same arrays, past one staging stage of rows too."""
    from mvector import _lib as L
    from mvector.audio import AudioSegment, PcmSegment
    p = preds[0]
    rng = np.random.default_rng(41)
    paths, arrays, rates = [], [], []
    for i in range(p.STAGE_ROWS + 5):
        rate = [16000, 44100, 8000, 48000][i % 4]
        data, arr = _file(_speech_like(rng, int(rng.integers(int(0.5 * rate), int(1.2 * rate))), 1 + i % 2), rate,
                          KINDS[i % len(KINDS)])
        q = tmp_path / f'p{i}.bin'
        q.write_bytes(data)
        paths.append(str(q))
        arrays.append(arr)
        rates.append(rate)
    ref_batch = p.predict_batch([AudioSegment(a, r) for a, r in zip(arrays, rates)])
    ref_one = p.predict(arrays[1], sample_rate=rates[1])

    def boom(*a, **k):
        raise AssertionError('host sample path used')
    monkeypatch.setattr(L.lib(), 'vp_host_stage_h2d', boom)
    monkeypatch.setattr(PcmSegment, 'samples', property(boom))
    assert np.array_equal(p.predict_batch(paths), ref_batch)
    assert np.array_equal(p.predict_batch([open(q, 'rb').read() for q in paths]), ref_batch)
    assert np.array_equal(p.predict(paths[1]), ref_one)


def test_mixed_list_of_pcm_flac_and_arrays(preds):
    from mvector.audio import AudioSegment, pcm_to_mono
    p = preds[1]
    rng = np.random.default_rng(43)
    items, arrays, rates = [], [], []
    for i in range(9):
        rate = [16000, 44100, 8000][i % 3]
        ints = _speech_like(rng, int(rate * 0.8), 1 + i % 2)
        if i % 3 == 0:
            data, arr = _file(ints, rate, KINDS[i % len(KINDS)])
            items.append(data)
        elif i % 3 == 1:
            data = fw.encode(ints, rate, 16, blocksize=4096, sub=lambda fi, c, x: dict(kind='fixed', order=2))
            arr = pcm_to_mono(ints.reshape(-1), ints.shape[1], 16)
            items.append(data)
        else:
            arr = pcm_to_mono(ints.reshape(-1), ints.shape[1], 16)
            items.append(AudioSegment(arr, rate))
        arrays.append(arr)
        rates.append(rate)
    assert np.array_equal(p.predict_batch(items), p.predict_batch([AudioSegment(a, r) for a, r in zip(arrays, rates)]))


def test_trainer_condition_converts_on_device(eng):
    from mvector.audio import AudioSegment
    from mvector.trainer import MVectorTrainer
    rng = np.random.default_rng(31)
    for k, (rate, ch) in enumerate(((16000, 1), (44100, 2), (8000, 3), (48000, 8))):
        data, arr = _file(_speech_like(rng, int(1.3 * rate), ch), rate, KINDS[k])
        for db in (None, -20):
            got = MVectorTrainer._condition(AudioSegment.from_bytes(data), 16000, db, 1.0, eng)
            ref = MVectorTrainer._condition(AudioSegment(arr, rate), 16000, db, 1.0, eng)
            assert np.array_equal(got.cpu().numpy(), ref.cpu().numpy()), (rate, ch, db)


def _recording_int16(sr):
    t = np.arange(sr * 4) / float(sr)

    def voice(f0, seed):
        v = sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 9))
        return 0.1 * v + 0.01 * np.random.RandomState(seed).randn(t.size)
    gap = np.zeros(sr // 2)
    x = np.concatenate([gap, voice(110.0, 1), gap, voice(290.0, 2), gap, voice(110.0, 3), gap])
    return np.round(x * 32767).astype(np.int64)[:, None]


@pytest.mark.parametrize('kind', ['s24le', 'ulaw', 's16be'])
def test_speaker_diarization_of_a_pcm_recording(preds, tmp_path, kind):
    p = preds[0]
    data, arr = _file(_recording_int16(16000), 16000, kind)
    path = tmp_path / 'rec.bin'
    path.write_bytes(data)
    got = p.speaker_diarization(str(path), sample_rate=16000, speaker_num=2)
    assert got == p.speaker_diarization(arr, sample_rate=16000, speaker_num=2)
    assert len(got) >= 3


def _wav16(path, ints, sr):
    with wave.open(str(path), 'wb') as w:
        w.setnchannels(ints.shape[1]); w.setsampwidth(2); w.setframerate(sr)
        w.writeframes(ints.astype('<i2').tobytes())


def test_evaluate_and_extract_features_equal_16_bit_wav(tmp_path, monkeypatch):
    """The same integers as 24-bit WAV, float32 WAV, 16-bit AIFF and mu-law WAV (its expansion), and as 16-bit WAV
    from the standard library read by the ``wave`` reader with host samples (the path such files took before PcmSegment,
    so the reference does not go through the conversion under test): identical (eer, min_dcf, threshold) and identical
    .npy features."""
    from mvector.audio import AudioSegment
    from mvector.trainer import MVectorTrainer
    from oracle import models as om
    rng = np.random.default_rng(51)
    rows = []
    for i in range(8):
        rate = [16000, 44100][i % 2]
        ints = _speech_like(rng, int(rate * (0.8 + 0.3 * i)), 1 + i % 2)
        kind = ('s24le', 'f32le', 's16be', 'ulaw')[i % 4]
        if kind == 'ulaw':                                   # the 16-bit values a mu-law file holds
            order = np.argsort(_MU)
            ints = _MU[order][np.clip(np.searchsorted(_MU[order], ints), 0, 255)]
        rows.append((ints, rate, kind))
    lists = {}
    for fmt in ('pcm', 'wav16'):
        (tmp_path / fmt).mkdir()
        lines = []
        for i, (ints, rate, kind) in enumerate(rows):
            path = tmp_path / fmt / f'{i}.bin'
            if fmt == 'pcm':
                path.write_bytes(_file(ints, rate, kind)[0])
            else:
                _wav16(path, ints, rate)
            lines.append(f'{path}\t{i % 4}\n')
        lists[fmt] = tmp_path / fmt / 'list.txt'
        lists[fmt].write_text(''.join(lines))
    results, feats = {}, {}
    for fmt in ('pcm', 'wav16'):
        if fmt == 'wav16':
            monkeypatch.setattr(AudioSegment, 'from_file', classmethod(lambda cls, f: AudioSegment._from_wave(f)))
        cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                            'use_dB_normalization': True, 'target_dB': -20},
                                'eval_conf': {'batch_size': 3, 'max_duration': 2}, 'train_list': str(lists[fmt]),
                                'enroll_list': str(lists[fmt]), 'trials_list': str(lists[fmt])},
               'preprocess_conf': {'feature_method': 'Fbank', 'method_args': dict(FARGS)},
               'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(MARGS)}}
        tr = MVectorTrainer(cfg, use_gpu=True)
        tr._setup_eval()
        tr.model.load_state_dict(om.random_state_dict('EcapaTdnn', 80, seed=5, **MARGS))
        results[fmt] = tr.evaluate()
        tr.extract_features(save_dir=str(tmp_path / fmt / 'features'), max_duration=1.5)
        out = (tmp_path / fmt / 'list_features.txt').read_text().splitlines()
        feats[fmt] = [np.load(ln.split('\t')[0]) for ln in out]
    assert results['pcm'] == results['wav16']
    assert len(feats['pcm']) == len(feats['wav16']) == 8
    for a, b in zip(feats['pcm'], feats['wav16']):
        assert np.array_equal(a, b)
