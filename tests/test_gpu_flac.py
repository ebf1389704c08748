"""Device FLAC decoding (csrc/flac.cu through Engine.decode_flac) against the plain Python decoder of the tests
(flac_oracle.py) followed by the shared integer -> float32 mono conversion (audio.pcm_to_mono), and the callers that
read FLAC: predict, predict_batch and contrast give the embeddings of the same audio passed as float32 arrays."""
import io
import os
import tempfile

import numpy as np
import pytest

import flac_cases
import flac_oracle as fo
import flac_writer as fw

pytestmark = pytest.mark.gpu

MARGS = dict(embd_dim=192, pooling_type='ASP', channels=[128, 128, 128, 128, 384], attention_channels=64,
             res2net_scale=4, se_channels=32)
FARGS = dict(sample_frequency=16000, num_mel_bins=80)


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    return Engine(0)


def _expected(data):
    from mvector.audio import pcm_to_mono
    ints, info = fo.decode(data)
    return pcm_to_mono(ints.reshape(-1), info['ch'], info['bps'])


def test_matrix_bit_identical_to_oracle(eng):
    cases = flac_cases.matrix()
    rows, status = eng.decode_flac([d for _, d, _, _ in cases], names=[n for n, _, _, _ in cases])
    rows, status = rows.cpu().numpy(), status.cpu().numpy()
    assert not status.any()
    for i, (name, data, pcm, bps) in enumerate(cases):
        ref = _expected(data)
        assert np.array_equal(rows[i, :ref.size].view(np.int32), ref.view(np.int32)), name
        assert not rows[i, ref.size:].any(), name                       # zero padding
    again, _ = eng.decode_flac([d for _, d, _, _ in cases])
    assert np.array_equal(again.cpu().numpy(), rows)


def test_long_constant_row(eng):
    """A row of 2^27 samples: 2048 CONSTANT frames of 65535 samples and one of 2048."""
    n = 1 << 27
    bs = 65535
    blocks = [bs] * (n // bs) + [n % bs]
    frames = []
    si = dict(rate=16000, bps=16)
    for fi, b in enumerate(blocks):
        w = fw.BitWriter()
        w.bits.extend(np.unpackbits(np.frombuffer(fw.frame_header(b, fi * bs, fi, 0, 0, si), np.uint8)).tolist())
        fw.write_subframe(w, [fi % 200 - 100] * 1, 16, kind='constant')
        w.align()
        body = w.bytes()
        frames.append(body + fw.crc16(body).to_bytes(2, 'big'))
    meta = b'fLaC' + bytes([0x80, 0, 0, 34]) + fw._streaminfo(bs, bs, 0, 0, 16000, 1, 16, n)
    data = meta + b''.join(frames)
    rows, status = eng.decode_flac([data])
    row = rows[0]
    assert row.numel() == n
    expect = np.repeat((np.arange(len(blocks)) % 200 - 100).astype(np.float32) / np.float32(32768), blocks)
    assert np.array_equal(row.cpu().numpy(), expect)


def _corrupt_cases(rng):
    pcm = fw.random_pcm(rng, 3000, 1, 16)
    good = fw.encode(pcm, 16000, 16, blocksize=512)
    from mvector.flac import parse_streaminfo
    fo_ = parse_streaminfo(good).frame_offset
    second = good.index(b'\xff\xf8', fo_ + 2)
    hdr_flip = bytearray(good); hdr_flip[second + 2] ^= 0x01          # the second frame's rate code
    pay_flip = bytearray(good); pay_flip[fo_ + 40] ^= 0x10
    truncated = good[:-50]
    contradict = bytearray(good)                             # STREAMINFO says 44.1 kHz; the frames say 16 kHz
    v = int.from_bytes(contradict[8 + 10:8 + 18], 'big')
    v = (v & ((1 << 44) - 1)) | (44100 << 44)
    contradict[8 + 10:8 + 18] = v.to_bytes(8, 'big')
    count = bytearray(good)                                  # STREAMINFO total one sample more than the frames hold
    v = int.from_bytes(count[8 + 10:8 + 18], 'big') + 1
    count[8 + 10:8 + 18] = v.to_bytes(8, 'big')
    return good, [bytes(hdr_flip), bytes(pay_flip), truncated, bytes(contradict), bytes(count)]


def test_malformed_streams_refused_others_exact(eng):
    rng = np.random.default_rng(3)
    good, bad = _corrupt_cases(rng)
    streams = [good] + bad + [good]
    names = ['good-a', 'header-bit', 'payload-bit', 'truncated', 'contradicts-streaminfo', 'sample-count', 'good-b']
    rows, status = eng.decode_flac(streams, names=names, check=False)
    st = status.cpu().numpy()
    assert st[0] == 0 and st[-1] == 0 and (st[1:-1] != 0).all(), st
    ref = _expected(good)
    r = rows.cpu().numpy()
    assert np.array_equal(r[0, :ref.size], ref) and np.array_equal(r[-1, :ref.size], ref)
    with pytest.raises(ValueError, match='payload-bit'):
        eng.decode_flac(streams, names=names)


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


@pytest.mark.parametrize('db', [0, 1])
def test_predict_from_flac_equals_arrays(preds, db, tmp_path):
    from mvector.audio import AudioSegment
    p = preds[db]
    rng = np.random.default_rng(11 + db)
    items, arrays, rates = [], [], []
    for i, rate in enumerate([8000, 16000, 44100, 48000] * 3):
        n = int(rng.integers(int(0.4 * rate), int(1.6 * rate)))
        ch = 1 + i % 2
        pcm = _speech_like(rng, n, ch)
        data = fw.encode(pcm, rate, 16, blocksize=1152, assign=(lambda fi: 10) if ch == 2 else None,
                         sub=lambda fi, c, x: dict(kind='fixed', order=2, part_order=2 if len(x) % 4 == 0 else 0))
        path = tmp_path / f'{i}.flac'
        path.write_bytes(data)
        kind = i % 3
        items.append(str(path) if kind == 0 else data if kind == 1 else open(path, 'rb'))
        arrays.append(_expected(data))
        rates.append(rate)
    got = p.predict_batch(items)
    ref = p.predict_batch([AudioSegment(a, r) for a, r in zip(arrays, rates)])
    assert np.array_equal(got, ref)
    for k in (0, 3, 5):
        path = str(tmp_path / f'{k}.flac')
        assert np.array_equal(p.predict(path), p.predict(arrays[k], sample_rate=rates[k]))
        assert np.array_equal(p.predict(io.BufferedReader(io.FileIO(path))), p.predict(arrays[k], sample_rate=rates[k]))
    c = p.contrast(str(tmp_path / '1.flac'), str(tmp_path / '2.flac'))
    f1, f2 = p.predict(arrays[1], sample_rate=rates[1]), p.predict(arrays[2], sample_rate=rates[2])
    assert c == np.dot(f1, f2) / (np.linalg.norm(f1) * np.linalg.norm(f2))
    seg = AudioSegment.from_file(str(tmp_path / '4.flac'))
    assert seg.duration == len(arrays[4]) / rates[4]


def test_predict_batch_more_than_stage_rows(preds):
    p = preds[1]
    rng = np.random.default_rng(21)
    n_items = p.STAGE_ROWS + 5
    datas, arrays = [], []
    for i in range(n_items):
        pcm = _speech_like(rng, int(rng.integers(5000, 9000)), 1)
        d = fw.encode(pcm, 16000, 16, blocksize=4096, sub=lambda fi, c, x: dict(kind='fixed', order=2))
        datas.append(d)
        arrays.append(_expected(d))
    assert np.array_equal(p.predict_batch(datas), p.predict_batch(arrays))


def test_trainer_condition_decodes_on_device(eng):
    """evaluate / extract_features condition a FLAC file from its device decode: the same row as the decoded array."""
    from mvector.audio import AudioSegment
    from mvector.trainer import MVectorTrainer
    rng = np.random.default_rng(31)
    for rate, ch in ((16000, 1), (44100, 2), (8000, 3)):
        data = fw.encode(_speech_like(rng, int(1.3 * rate), ch), rate, 16, blocksize=4096,
                         sub=lambda fi, c, x: dict(kind='fixed', order=2))
        for db in (None, -20):
            got = MVectorTrainer._condition(AudioSegment.from_bytes(data), 16000, db, 1.0, eng)
            ref = MVectorTrainer._condition(AudioSegment(_expected(data), rate), 16000, db, 1.0, eng)
            assert np.array_equal(got.cpu().numpy(), ref.cpu().numpy()), (rate, ch, db)


# ------------------------------------------------------------------------------------------------ the FLAC-only path
def _flac_files(tmp_path, rng, rates, prefix='f'):
    paths, arrays = [], []
    for i, rate in enumerate(rates):
        pcm = _speech_like(rng, int(rng.integers(int(0.5 * rate), int(1.5 * rate))), 1 + i % 2)
        data = fw.encode(pcm, rate, 16, blocksize=4096, sub=lambda fi, c, x: dict(kind='fixed', order=2))
        p = tmp_path / f'{prefix}{i}.flac'
        p.write_bytes(data)
        paths.append(str(p))
        arrays.append(_expected(data))
    return paths, arrays


def test_flac_only_call_decodes_into_the_staging_slots(preds, tmp_path, monkeypatch):
    """A call whose items are all FLAC never stages host PCM (vp_host_stage_h2d) and never reads FlacSegment.samples;
    its embeddings are those of the decoded arrays."""
    from mvector import _lib as L
    from mvector.audio import AudioSegment, FlacSegment
    p = preds[0]
    rng = np.random.default_rng(41)
    rates = [16000, 44100, 8000, 48000, 16000]
    paths, arrays = _flac_files(tmp_path, rng, rates)
    ref_batch = p.predict_batch([AudioSegment(a, r) for a, r in zip(arrays, rates)])
    ref_one = p.predict(arrays[1], sample_rate=rates[1])

    def boom(*a, **k):
        raise AssertionError('host PCM path used')
    monkeypatch.setattr(L.lib(), 'vp_host_stage_h2d', boom)
    monkeypatch.setattr(FlacSegment, 'samples', property(boom))
    assert np.array_equal(p.predict_batch(paths), ref_batch)
    assert np.array_equal(p.predict_batch([open(q, 'rb').read() for q in paths]), ref_batch)
    assert np.array_equal(p.predict(paths[1]), ref_one)


def test_refused_stream_in_a_batch_names_the_file(preds, tmp_path):
    p = preds[1]
    rng = np.random.default_rng(42)
    paths, _ = _flac_files(tmp_path, rng, [16000, 16000, 16000])
    bad = bytearray(open(paths[1], 'rb').read())
    bad[len(bad) // 2] ^= 0x40
    open(paths[1], 'wb').write(bytes(bad))
    with pytest.raises(ValueError, match='f1.flac'):
        p.predict_batch(paths)


def test_batch_past_2_31_bytes(eng):
    """33 copies of one 2^25-sample 16-bit verbatim stream: 2.2 GB of concatenated bytes, every row exact."""
    import torch
    n, bs = 1 << 25, 65535
    x = np.random.default_rng(5).integers(-32768, 32768, size=n, dtype=np.int64)
    nfr = -(-n // bs)
    si = dict(rate=16000, bps=16)
    heads = [fw.frame_header(min(bs, n - f * bs), f * bs, f, 0, 0, si) for f in range(nfr)]
    bodies = []
    be = x.astype('>i2').view(np.uint8)
    for f in range(nfr):
        lo, hi = f * bs, min(n, (f + 1) * bs)
        bodies.append(np.concatenate([np.frombuffer(heads[f], np.uint8), np.array([0x02], np.uint8), be[2 * lo:2 * hi]]))
    crcs = _crc16_many(bodies)
    frames = b''.join(b.tobytes() + int(c).to_bytes(2, 'big') for b, c in zip(bodies, crcs))
    data = b'fLaC' + bytes([0x80, 0, 0, 34]) + fw._streaminfo(bs, bs, 0, 0, 16000, 1, 16, n) + frames
    copies = 33
    assert copies * len(data) > 2 ** 31
    rows, status = eng.decode_flac([data] * copies)
    expect = torch.from_numpy(x.astype(np.float32) / np.float32(32768)).to(rows.device)
    for r in range(copies):
        assert torch.equal(rows[r], expect), r


def _crc16_many(bodies):
    """CRC-16 of many byte strings at once (table driven, vectorised over the strings)."""
    tab = np.array([fw.crc16(bytes([i])) for i in range(256)], dtype=np.uint32)
    L = max(len(b) for b in bodies)
    lens = np.array([len(b) for b in bodies])
    mat = np.zeros((len(bodies), L), dtype=np.uint32)
    for i, b in enumerate(bodies):
        mat[i, L - len(b):] = b                     # leading zeros leave a CRC with zero initial value unchanged
    c = np.zeros(len(bodies), dtype=np.uint32)
    for k in range(L):
        c = ((c << 8) & 0xFFFF) ^ tab[((c >> 8) ^ mat[:, k]) & 0xFF]
    assert (lens > 0).all()
    return c


# ------------------------------------------------------------------------------------------------ other callers
def _recording_int16(sr):
    t = np.arange(sr * 4) / float(sr)

    def voice(f0, seed):
        v = sum(np.sin(2 * np.pi * f0 * h * t) / h for h in range(1, 9))
        return 0.1 * v + 0.01 * np.random.RandomState(seed).randn(t.size)
    gap = np.zeros(sr // 2)
    x = np.concatenate([gap, voice(110.0, 1), gap, voice(290.0, 2), gap, voice(110.0, 3), gap])
    return np.round(x * 32767).astype(np.int64)


def test_speaker_diarization_of_a_flac_recording(preds, tmp_path):
    p = preds[0]
    pcm = _recording_int16(16000)
    data = fw.encode(pcm, 16000, 16, blocksize=4096, sub=lambda fi, c, x: dict(kind='fixed', order=2))
    path = tmp_path / 'rec.flac'
    path.write_bytes(data)
    got = p.speaker_diarization(str(path), sample_rate=16000, speaker_num=2)
    assert got == p.speaker_diarization(_expected(data), sample_rate=16000, speaker_num=2)
    assert len(got) >= 3


def _wav16(path, pcm, sr):
    import wave
    with wave.open(str(path), 'wb') as w:
        w.setnchannels(pcm.shape[1]); w.setsampwidth(2); w.setframerate(sr)
        w.writeframes(pcm.astype('<i2').tobytes())
    return str(path)


def test_evaluate_and_extract_features_flac_equal_wav(tmp_path):
    """The same integers as FLAC and as 16-bit WAV: identical (eer, min_dcf, threshold) and identical .npy features; a
    corrupt file is replaced by its successor in either format."""
    from mvector.trainer import MVectorTrainer
    from oracle import models as om
    rng = np.random.default_rng(51)
    lists = {}
    for fmt in ('flac', 'wav'):
        (tmp_path / fmt).mkdir()
    rows = []
    for i in range(8):
        rate = [16000, 44100][i % 2]
        pcm = _speech_like(rng, int(rate * (0.8 + 0.3 * i)), 1 + i % 2)
        rows.append((pcm, rate))
    for fmt in ('flac', 'wav'):
        lines = []
        for i, (pcm, rate) in enumerate(rows):
            p = tmp_path / fmt / f'{i}.{fmt}'
            if fmt == 'flac':
                p.write_bytes(fw.encode(pcm, rate, 16, blocksize=4096, sub=lambda fi, c, x: dict(kind='fixed', order=2)))
            else:
                _wav16(p, pcm, rate)
            lines.append(f'{p}\t{i % 4}\n')
        lists[fmt] = tmp_path / fmt / 'list.txt'
        lists[fmt].write_text(''.join(lines))
    results, feats = {}, {}
    for fmt in ('flac', 'wav'):
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
        # a corrupt file 2 in both formats: extract_features logs it and takes file 3 in its place
        bad = tmp_path / fmt / f'2.{fmt}'
        raw = bytearray(bad.read_bytes())
        if fmt == 'flac':
            raw[len(raw) // 2] ^= 0x40
        else:
            raw[:4] = b'JUNK'
        bad.write_bytes(bytes(raw))
        tr.extract_features(save_dir=str(tmp_path / fmt / 'features'), max_duration=1.5)
        out = (tmp_path / fmt / 'list_features.txt').read_text().splitlines()
        feats[fmt] = [np.load(ln.split('\t')[0]) for ln in out]
    assert results['flac'] == results['wav']
    assert len(feats['flac']) == len(feats['wav']) == 8
    for a, b in zip(feats['flac'], feats['wav']):
        assert np.array_equal(a, b)
    assert np.array_equal(feats['flac'][2], feats['flac'][3])


def test_register_and_recognition_with_a_flac_audio_db(tmp_path):
    import torch
    from mvector.predict import MVectorPredictor
    from oracle import models as om
    rng = np.random.default_rng(61)
    sd = om.random_state_dict('EcapaTdnn', 80, seed=5, **MARGS)
    md = tmp_path / 'model'
    md.mkdir()
    torch.save({'0.' + k: v for k, v in sd.items()}, str(md / 'model.pth'))
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': True, 'target_dB': -20},
                            'eval_conf': {'batch_size': 4, 'max_duration': 20}},
           'preprocess_conf': {'use_hf_model': False, 'feature_method': 'Fbank', 'method_args': dict(FARGS)},
           'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(MARGS)}}
    spk = [(_speech_like(rng, 20000, 1), 16000) for _ in range(6)]
    feats = {}
    for fmt in ('flac', 'wav'):
        db = tmp_path / f'db_{fmt}'
        for i, (pcm, rate) in enumerate(spk[:5]):
            d = db / f'user{i % 3}'
            d.mkdir(parents=True, exist_ok=True)
            if fmt == 'flac':
                (d / f'{i}.flac').write_bytes(fw.encode(pcm, rate, 16, blocksize=4096))
            else:
                _wav16(d / f'{i}.wav', pcm, rate)
        pred = MVectorPredictor(configs=cfg, audio_db_path=str(db), model_path=str(md), use_gpu=True)
        feats[fmt] = {(nm, os.path.splitext(os.path.basename(pth))[0]): f
                      for nm, pth, f in zip(pred.users_name, pred.users_audio_path, pred.audio_feature)}
        probe = tmp_path / f'probe.{fmt}'
        if fmt == 'flac':
            probe.write_bytes(fw.encode(spk[5][0], 16000, 16, blocksize=4096))
        else:
            _wav16(probe, spk[5][0], 16000)
        assert pred.register(str(probe), 'newcomer')[0]
        name, score = pred.recognition(str(probe), threshold=0.5)
        assert name == 'newcomer', (fmt, name, score)
    assert sorted(feats['flac']) == sorted(feats['wav']) and len(feats['flac']) == 5
    for k in feats['flac']:
        assert np.array_equal(feats['flac'][k], feats['wav'][k]), k
