"""The ragged front-end (vp_features_each through AudioFeaturizer.forward_each) against one-row calls, and evaluate /
extract_features, which run it a group of files at a time, against the file-by-file loop they replace: bit for bit."""
import wave

import numpy as np
import pytest
import torch

import flac_writer as fw
import pcm_writer as pw

pytestmark = pytest.mark.gpu

CONFIGS = [
    ('Fbank', dict(sample_frequency=16000, num_mel_bins=80)),
    ('Fbank', dict(sample_frequency=16000, num_mel_bins=80, snip_edges=False)),
    ('MelSpectrogram', dict(sample_rate=16000, n_fft=512, hop_length=160, win_length=400, n_mels=64)),
    ('MelSpectrogram', dict(sample_rate=16000, n_fft=512, hop_length=160, n_mels=64, center=False, pad=3)),
    ('Spectrogram', dict(n_fft=400, hop_length=160, normalized=True)),
    ('MFCC', dict(sample_rate=16000, n_mfcc=40, melkwargs=dict(n_fft=512, hop_length=160, n_mels=64))),
    ('MFCC', dict(sample_rate=16000, n_mfcc=40, log_mels=True, melkwargs=dict(n_fft=512, hop_length=160, n_mels=64))),
]
MARGS = dict(embd_dim=192, pooling_type='ASP', channels=[128, 128, 128, 128, 384], attention_channels=64,
             res2net_scale=4, se_channels=32)


def _valid(fz, n):
    """Whether a one-row call takes n samples (the library's own check, no launch)."""
    import ctypes as C
    from mvector import _lib as L
    info = (C.c_int32 * 8)()
    return L.lib().vp_frontend_plan_info(fz.engine.handle, 1, n, fz.feat_fun.desc.post, info) == L.VP_OK


def _samples_for(fz, T):
    """The fewest samples a one-row call takes with exactly T frames (None when even the shortest row has more), moved
    off a multiple of the hop where that keeps T."""
    for n in range(1, 1 << 20):
        if _valid(fz, n) and fz.num_frames(n) >= T:
            if fz.num_frames(n) > T:
                return None
            return n + 1 if n % fz.feat_fun.hop == 0 and fz.num_frames(n + 1) == T else n


def _one(fz, x):
    return fz(torch.from_numpy(x).cuda()).squeeze(0).cpu().numpy()


def _check_rows(fz, rows, ld):
    w = np.zeros((len(rows), ld), dtype=np.float32)
    for i, r in enumerate(rows):
        w[i, :r.size] = r
    feats, tb = fz.forward_each(torch.from_numpy(w).cuda(), [r.size for r in rows])
    got = feats.cpu().numpy()
    assert got.shape[1] == tb.max()
    for i, r in enumerate(rows):
        ref = _one(fz, r)
        assert tb[i] == ref.shape[0] == fz.num_frames(r.size)
        assert np.array_equal(got[i, :tb[i]], ref), (i, r.size)
        tail = got[i, tb[i]:]
        assert not tail.any() and not np.signbit(tail).any(), i         # +0.0 padding
    return got


@pytest.mark.parametrize('method,args', CONFIGS, ids=[f'{m}-{i}' for i, (m, _) in enumerate(CONFIGS)])
def test_each_row_equals_its_one_row_call(method, args):
    from mvector.data_utils.featurizer import AudioFeaturizer
    fz = AudioFeaturizer(method, method_args=args)
    rng = np.random.default_rng(7)
    lens = [n for n in (_samples_for(fz, T) for T in (1, 15, 16, 17, 64, 65)) if n is not None]
    assert len(lens) >= 5
    lens.append(lens[2] + 37)                           # not a multiple of the hop
    long_n = 160003                                     # about 10 s
    ld = long_n + 11                                    # one row of exactly ld samples
    lens = lens[:2] + [long_n] + lens[2:4] + [ld] + lens[4:]     # the shortest first, the longest inside
    rows = [(rng.standard_normal(n) * rng.uniform(0.01, 0.5)).astype(np.float32) for n in lens]
    _check_rows(fz, rows, ld)


def test_mfcc_rows_clamp_against_their_own_maximum():
    from mvector.data_utils.featurizer import AudioFeaturizer
    fz = AudioFeaturizer('MFCC', method_args=CONFIGS[5][1])
    rng = np.random.default_rng(8)
    ld = 16000
    rows = [(rng.standard_normal(ld) * a).astype(np.float32) for a in (1e-5, 1.0, 1e-5)]
    got = _check_rows(fz, rows, ld)
    # Rows of one length frame and mean-normalise the same alone as in one vp_features call over the batch, so the only
    # difference left is the clamp: the batch call clamps every row against the loud row's maximum.
    w = np.zeros((3, ld), dtype=np.float32)
    for i, r in enumerate(rows):
        w[i, :r.size] = r
    whole = fz.forward_keep(torch.from_numpy(w).cuda()).cpu().numpy()
    assert np.array_equal(whole[1], got[1])
    assert not np.array_equal(whole[0], got[0]) and not np.array_equal(whole[2], got[2])


# ---------------------------------------------------------------------------------------------- evaluate / extract
def _speech(rng, n, ch=1):
    t = np.arange(n)
    x = 0.3 * np.sin(2 * np.pi * rng.uniform(100, 400) * t / 16000.0) + 0.05 * rng.standard_normal(n)
    x = np.clip(x * 32767, -32768, 32767).astype(np.int64)
    return np.repeat(x[:, None], ch, axis=1)


def _write_list(tmp_path, seed, extra=()):
    rng = np.random.default_rng(seed)
    lines = []
    kinds = ['wav16', 'wav24', 'flac', 'wave10']
    for i in range(40):
        rate = 16000 if i % 3 else 44100
        n = int(rng.uniform(0.5, 6.0) * rate)
        kind = kinds[i % 4]
        p = tmp_path / f'u{i}.{"flac" if kind == "flac" else "wav"}'
        if kind == 'wav16':
            p.write_bytes(pw.wav(pw.encode(_speech(rng, n).reshape(-1), 's16le'), rate, 1, 's16le'))
        elif kind == 'wav24':
            pcm = _speech(rng, n).reshape(-1) * 256 + rng.integers(0, 256, n)
            p.write_bytes(pw.wav(pw.encode(pcm, 's24le'), rate, 1, 's24le'))
        elif kind == 'flac':
            ch = 1 + i % 2
            p.write_bytes(fw.encode(_speech(rng, n, ch), rate, 16, blocksize=4096,
                                    sub=lambda fi, c, x: dict(kind='fixed', order=2)))
        else:                                           # ten channels: the PCM parser refuses, the wave reader reads it
            with wave.open(str(p), 'wb') as w:
                w.setnchannels(10); w.setsampwidth(2); w.setframerate(rate)
                w.writeframes(_speech(rng, n, 10).astype('<i2').tobytes())
        lines.append(f'{p}\t{i % 7}\n')
    lines.extend(extra)
    lst = tmp_path / 'list.txt'
    lst.write_text(''.join(lines))
    return str(lst), lines


def _trainer(lst, method, args, max_duration=2, bs=3):
    from mvector.trainer import MVectorTrainer
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.6, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': True, 'target_dB': -20},
                            'eval_conf': {'batch_size': bs, 'max_duration': max_duration}, 'train_list': lst,
                            'enroll_list': lst, 'trials_list': lst},
           'preprocess_conf': {'feature_method': method, 'method_args': dict(args)},
           'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(MARGS)}}
    return MVectorTrainer(cfg, use_gpu=True)


def _per_file_embeddings(tr, lst):
    entries = tr._eval_order(lst)
    bs = tr.configs.dataset_conf.eval_conf.batch_size
    out = []
    for s in range(0, len(entries), bs):
        items = [tr._eval_feature(p) for p, _ in entries[s:s + bs]]
        out.append(tr.model(tr._zero_pad_features(items)).cpu().numpy())
    return np.concatenate(out)


@pytest.mark.parametrize('method,args', [CONFIGS[0], CONFIGS[5]], ids=['Fbank', 'MFCC'])
def test_evaluate_equals_the_per_file_loop(tmp_path, method, args, monkeypatch):
    from mvector import _lib as L
    from mvector.trainer import MVectorTrainer
    from oracle import models as om
    lst, _ = _write_list(tmp_path, 3)
    tr = _trainer(lst, method, args)
    tr._setup_eval()
    F = tr.audio_featurizer.feature_dim
    tr.model.load_state_dict(om.random_state_dict('EcapaTdnn', F, seed=5, **MARGS))
    tr.model.eval()
    ref = _per_file_embeddings(tr, lst)
    monkeypatch.setattr(MVectorTrainer, 'MAX_GROUP', 7)          # 6 files a group: several groups
    lib = L.lib()
    calls = []
    for name in ('vp_flac_decode', 'vp_pcm_decode', 'vp_resample', 'vp_gain_normalize', 'vp_features_each',
                 'vp_features'):
        real = getattr(lib, name)
        monkeypatch.setattr(lib, name, lambda *a, _n=name, _r=real: calls.append(_n) or _r(*a))
    got, labels = tr._embed_list(lst)
    assert np.array_equal(got, ref)
    groups = -(-40 // 6)                                        # once per group, not once per file
    for name in ('vp_gain_normalize', 'vp_features_each'):
        assert calls.count(name) == groups, (name, calls.count(name))
    for name in ('vp_flac_decode', 'vp_pcm_decode', 'vp_resample'):
        assert 0 < calls.count(name) <= groups, (name, calls.count(name))
    assert 'vp_features' not in calls
    res = tr.evaluate()
    monkeypatch.setattr(MVectorTrainer, '_embed_list', lambda self, name: (_per_file_embeddings(self, name), labels))
    assert tr.evaluate() == res


def test_extract_features_equals_the_per_file_rule(tmp_path):
    from mvector.audio import AudioSegment, FlacSegment
    rng = np.random.default_rng(9)
    short = tmp_path / 'short.wav'
    short.write_bytes(pw.wav(pw.encode(_speech(rng, 4000).reshape(-1), 's16le'), 16000, 1, 's16le'))
    good = fw.encode(_speech(rng, 30000), 16000, 16, blocksize=1024, sub=lambda fi, c, x: dict(kind='fixed', order=2))
    bad = bytearray(good)
    bad[len(bad) // 2] ^= 0x40
    corrupt = tmp_path / 'corrupt.flac'
    corrupt.write_bytes(bytes(bad))
    extra = [f'{short}\t3\n', f'{corrupt}\t4\n']
    lst, lines = _write_list(tmp_path, 4, extra)
    lines = [f'{corrupt}\t5\n'] + lines                        # the corrupt file also first: its successor serves it
    (tmp_path / 'list.txt').write_text(''.join(lines))
    tr = _trainer(lst, *CONFIGS[0])
    tr.extract_features(save_dir=str(tmp_path / 'features'), max_duration=2.5)
    out = (tmp_path / 'list_features.txt').read_text().splitlines()
    assert len(out) == len(lines)
    eng = tr.audio_featurizer.engine
    paths = [ln.split('\t')[0] for ln in lines]

    def source(idx):                                   # the per-file rule: successors, each FLAC decoded in turn
        j = idx
        while True:
            try:
                cand = AudioSegment.from_file(paths[j])
                if cand.duration >= 0.6:
                    if isinstance(cand, FlacSegment):
                        cand.decode_device(eng)
                    return j
            except Exception:  # noqa: BLE001
                pass
            j = (j + 1) % len(paths)

    for idx, ln in enumerate(out):
        j = source(idx)
        assert paths[j] not in (str(short), str(corrupt))
        seg = AudioSegment.from_file(paths[j])
        ref = tr.audio_featurizer(tr._condition(seg, 16000, -20, 2.5, eng)).squeeze(0).cpu().numpy()
        path, label = ln.split('\t')
        assert int(label) == int(lines[j].split('\t')[1]), idx
        assert np.array_equal(np.load(path), ref), idx
