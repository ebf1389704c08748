"""HF wav2vec 2.0 / WavLM front-end on the GPU (vp_frontend_set_hf): features and EcapaTdnn embeddings against the
reference's golden, the device normalisation bit for bit against numpy, row independence bit for bit, the length
rule, and every caller built on the featurizer with a `use_hf_model` config."""
import ctypes as C
import json
import os
import sys
import tempfile
import wave

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, rel_l2

sys.path.insert(0, os.path.join(ROOT, 'tests'))
from hf_writer import write_hf_dir  # noqa: E402

pytestmark = pytest.mark.gpu

# Feature parity, as for Fbank (test_gpu_parity.py): the reference's own fp32 stack is not the exact value of its
# formula either (a few 1e-6 away on these cases), so the tests check
#   (1) |ours - exact| <= FEAT_TOL          (exact: tests/hf_oracle.py in fp64 from the processor's float32 output)
#   (2) |ours - reference| <= |reference - exact| + FEAT_TOL   (on the channels the golden file stores)
FEAT_TOL = 1e-4
EMB_TOL = 1e-4
CASES = ['small_group', 'small_group_raw', 'small_layer', 'small_layer_raw', 'base_1s', 'base_3s']


@pytest.fixture(scope='module')
def golden():
    z = np.load(os.path.join(GOLDEN, 'hf_frontend.npz'))
    return z, json.loads(bytes(z['meta']).decode())


@pytest.fixture(scope='module')
def dirs(golden, tmp_path_factory):
    _, meta = golden
    out = {}
    for name, c in meta['cases'].items():
        d = str(tmp_path_factory.mktemp(name))
        kw = {k: (tuple(v) if isinstance(v, list) else v) for k, v in c['writer'].items()}
        write_hf_dir(d, **kw)
        out[name] = d
    return out


def _waves(meta, name):
    from hf_writer import seeded_waves
    c = meta['cases'][name]
    return seeded_waves(c['B'], c['L'], c['wave_seed'], c['ratio']), np.asarray(c['ratio'], np.float32)


def _fz(d):
    from mvector.data_utils.featurizer import AudioFeaturizer
    return AudioFeaturizer(feature_method=d, use_hf_model=True, method_args={'use_gpu': True})


def _model(F, seed, margs):
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object
    from oracle import models as om
    sd = om.random_state_dict('EcapaTdnn', F, seed=seed, **margs)
    m = build_model(F, dict_to_object({'model_conf': {'model': 'EcapaTdnn', 'model_args': margs}}))
    m.load_state_dict({'0.' + k: v for k, v in sd.items()})
    return m, sd


@pytest.mark.parametrize('name', CASES)
def test_features_and_embeddings_match_reference(golden, dirs, name):
    z, meta = golden
    fz = _fz(dirs[name])
    wave, ratio = _waves(meta, name)
    feats = fz(torch.from_numpy(wave), torch.from_numpy(ratio))
    step = meta['cases'][name]['feat_step']
    want = z[name + '/feats']                          # the reference's features, every step-th channel
    got = feats.cpu().numpy()
    assert got[:, :, ::step].shape == want.shape
    import hf_oracle
    from hf_writer import feature_weights
    kw = meta['cases'][name]['writer']
    sd = feature_weights(tuple(kw['conv_dim']), (10, 3, 3, 3, 3, 2, 2), kw['norm'], kw.get('conv_bias', False),
                         kw['seed'])
    exact = hf_oracle.featurize(wave, ratio, sd, kw['norm'], (10, 3, 3, 3, 3, 2, 2), (5, 2, 2, 2, 2, 2, 2),
                                kw.get('do_normalize', True), dtype=torch.float64).numpy()
    e_got = np.abs(got - exact).max()
    e_ref, d = np.abs(want - exact[:, :, ::step]).max(), np.abs(got[:, :, ::step] - want).max()
    print(f'{name}: |ours-exact| {e_got:.2e}  |ours-ref| {d:.2e}  |ref-exact| {e_ref:.2e}')
    assert e_got <= FEAT_TOL and d <= e_ref + FEAT_TOL
    m, _ = _model(got.shape[2], meta['cases'][name]['model_seed'], meta['margs'])
    emb = m(feats).cpu().numpy()
    assert rel_l2(emb, z[name + '/emb']).max() < EMB_TOL


def _scratch_rows(fz, w):
    """vp_features on w, returning its scratch: the call's first region holds the normalised rows, [rows of s_0
    samples, cp channels] per row (hf.cu, hf_normalize_kernel)."""
    from mvector import _lib as L
    h = fz.engine.handle
    lib = L.lib()
    B, n = w.shape
    feats = torch.empty(B, fz.num_frames(n), fz.feature_dim, device='cuda')
    sc = torch.zeros(int(lib.vp_frontend_scratch_floats(h, B, n)), device='cuda')
    assert lib.vp_features(h, C.c_void_p(w.data_ptr()), B, n, None, C.c_void_p(feats.data_ptr()),
                           C.c_void_p(sc.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    info = (C.c_int32 * 8)()
    assert lib.vp_frontend_plan_info(h, B, n, 0, info) == 0
    T0, kt, cp = info[2], info[5], info[6]
    R0 = T0 + kt - 1
    s0 = fz.feat_fun.ckpt.conv_stride[0]
    x = sc[:B * R0 * cp].view(B, R0, cp)[:, :, :s0].reshape(B, -1)
    return x.cpu().numpy()[:, :min(n, R0 * s0)]          # the samples the conv stack reads


@pytest.mark.parametrize('n', [400, 401, 405, 407, 512, 513, 1023, 1024, 1025, 2047, 2048, 2049, 4096, 4097, 16000,
                               16001, 48003, 65535, 65536, 65537])
def test_device_normalisation_is_numpy_bit_for_bit(dirs, n):
    fz = _fz(dirs['small_group'])
    rng = np.random.default_rng(n)
    w = (rng.standard_normal((3, n)) * np.array([[0.1], [3.0], [1e-3]]) + np.array([[0.0], [0.5], [-2.0]]))
    w = w.astype(np.float32)
    got = _scratch_rows(fz, torch.from_numpy(w).cuda())
    want = np.stack([(r - r.mean()) / np.sqrt(r.var() + 1e-7) for r in w])[:, :got.shape[1]]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_device_normalisation_short_and_zero_rows(dirs):
    """The pairwise tree below 8, at 128 / 129 and an all-zero row, through a one-layer stack that takes every length."""
    d = tempfile.mkdtemp()
    write_hf_dir(d, conv_dim=(16,), conv_kernel=(5,), conv_stride=(5,), seed=3)
    fz = _fz(d)
    for n in (5, 7, 8, 9, 15, 16, 17, 127, 128, 129, 130, 255, 256, 257, 1000):
        rng = np.random.default_rng(n)
        w = (rng.standard_normal((2, n)) * 0.2 + 0.1).astype(np.float32)
        w[1] = 0
        got = _scratch_rows(fz, torch.from_numpy(w).cuda())
        want = np.stack([(r - r.mean()) / np.sqrt(r.var() + 1e-7) for r in w])[:, :got.shape[1]]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), n


def test_raw_rows_pass_through(dirs):
    fz = _fz(dirs['small_group_raw'])
    w = (np.random.default_rng(1).standard_normal((2, 3001)) * 0.3).astype(np.float32)
    got = _scratch_rows(fz, torch.from_numpy(w).cuda())
    assert np.array_equal(got, w[:, :got.shape[1]])


@pytest.mark.parametrize('name', ['small_group', 'small_layer', 'base_1s'])
def test_rows_are_independent(dirs, name):
    """A padded-call row is the same bits whatever the other rows hold and however the batch is sliced; a ragged row
    is the same bits as a one-row call on its own samples."""
    fz = _fz(dirs[name])
    rng = np.random.default_rng(5)
    L = 12345
    w = torch.from_numpy((rng.standard_normal((5, L)) * 0.1).astype(np.float32)).cuda()
    ratio = torch.tensor([1.0, 0.5, 0.9, 0.3, 0.77])
    full = fz(w, ratio).cpu()
    w2 = w.clone()
    w2[[0, 2, 4]] = torch.randn(3, L, device='cuda') * 5
    other = fz(w2, ratio).cpu()
    assert torch.equal(full[[1, 3]], other[[1, 3]])
    for b in range(5):
        assert torch.equal(fz(w[b:b + 1], ratio[b:b + 1]).cpu()[0], full[b])
    assert torch.equal(torch.cat([fz(w[:2], ratio[:2]).cpu(), fz(w[2:], ratio[2:]).cpu()]), full)
    lens = [L, 6000, 11111, 400, 9000]
    feats, tb = fz.forward_each(w, lens)
    feats = feats.cpu()
    for b, n in enumerate(lens):
        one = fz(w[b:b + 1, :n].contiguous()).cpu()[0]
        assert tb[b] == one.shape[0]
        assert torch.equal(feats[b, :tb[b]], one)
        assert (feats[b, tb[b]:] == 0).all()


def test_slices_beyond_the_scratch_cap(dirs):
    """10 s rows at 512 channels: the call runs in several slices and every row equals its one-row call."""
    from mvector import _lib as L
    fz = _fz(dirs['base_1s'])
    B, n = 10, 160000
    info = (C.c_int32 * 8)()
    assert L.lib().vp_frontend_plan_info(fz.engine.handle, B, n, 0, info) == 0
    assert info[1] > 1, 'expected more than one slice'
    assert L.lib().vp_frontend_scratch_floats(fz.engine.handle, B, n) <= L.HF_SCRATCH_CAP
    w = torch.randn(B, n, device='cuda') * 0.1
    full = fz(w).cpu()
    for b in (0, info[0] - 1, info[0], B - 1):
        assert torch.equal(fz(w[b:b + 1]).cpu()[0], full[b])


def test_shortest_length(dirs):
    fz = _fz(dirs['base_1s'])
    w = torch.randn(2, 400, device='cuda')
    assert fz(w).shape == (2, 1, 512)
    with pytest.raises(RuntimeError, match='399 samples'):
        fz(w[:, :399].contiguous())
    with pytest.raises(RuntimeError, match='399 samples'):
        fz.forward_each(torch.randn(2, 1000, device='cuda'), [1000, 399])


# ------------------------------------------------------------------------------------------------ callers
def _cfg(d, margs, **ds):
    dataset = {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000, 'use_dB_normalization': False,
               'target_dB': -20}
    dataset.update(ds)
    return {'dataset_conf': {'dataset': dataset, 'eval_conf': {'batch_size': 4, 'max_duration': 20}},
            'preprocess_conf': {'use_hf_model': True, 'feature_method': d, 'method_args': {'use_gpu': True}},
            'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(margs)}}


_MODEL_DIR = []


@pytest.fixture(scope='module')
def predictor(golden, dirs, tmp_path_factory):
    from mvector.predict import MVectorPredictor
    z, meta = golden
    name = 'small_layer'
    _, sd = _model(48, meta['cases'][name]['model_seed'], meta['margs'])
    td = str(tmp_path_factory.mktemp('model'))
    _MODEL_DIR[:] = [td]
    torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
    return MVectorPredictor(configs=_cfg(dirs[name], meta['margs']), model_path=td, use_gpu=True), name


def _trimmed(z, name):
    w, r = _waves(json.loads(bytes(z['meta']).decode()), name)
    return [row[:int(round(float(x) * w.shape[1]))].copy() for row, x in zip(w, r)]


def test_predict_batch_and_predict(golden, predictor):
    z, _ = golden
    pred, name = predictor
    waves = _trimmed(z, name)
    emb = pred.predict_batch(waves)
    assert rel_l2(emb, z[name + '/emb']).max() < EMB_TOL
    one = pred.predict(waves[2])
    assert rel_l2(one, pred.predict_batch([waves[2]])[0]).max() < EMB_TOL
    s = pred.contrast(waves[0], waves[1])
    e0, e1 = pred.predict(waves[0]), pred.predict(waves[1])
    assert abs(s - float(np.dot(e0, e1) / np.linalg.norm(e0) / np.linalg.norm(e1))) < 1e-5


def test_register_recognition_and_db_load(golden, dirs, predictor, tmp_path):
    from mvector.predict import MVectorPredictor
    z, meta = golden
    pred, name = predictor
    waves = _trimmed(z, name)
    db = str(tmp_path / 'db')
    mk = lambda: MVectorPredictor(configs=_cfg(dirs[name], meta['margs']), audio_db_path=db, model_path=_MODEL_DIR[0],
                                  use_gpu=True, threshold=0.5)
    p1 = mk()
    assert p1.register(waves[0], 'alice')[0] and p1.register(waves[1], 'bob')[0]
    assert p1.recognition(waves[0])[0] == 'alice'
    p2 = mk()                                                      # the voiceprint DB read back at construction
    assert sorted(set(p2.get_users())) == ['alice', 'bob']
    assert p2.recognition(waves[1])[0] == 'bob'


def test_predict_batch_sharded_single_process(golden, predictor):
    from mvector.distributed import predict_batch_sharded
    z, _ = golden
    pred, name = predictor
    waves = _trimmed(z, name)
    got = predict_batch_sharded(pred, waves)
    assert np.array_equal(np.asarray(got), pred.predict_batch(waves))


def test_speaker_diarization_runs_on_hf_features(predictor):
    pred, _ = predictor
    assert pred._audio_featurizer.num_frames(24000) == 74
    rng = np.random.default_rng(2)
    t = np.arange(16000 * 6) / 16000.0
    a = 0.3 * np.sin(2 * np.pi * 180 * t) * (t < 3) + 0.3 * np.sin(2 * np.pi * 310 * t) * (t >= 3)
    a = (a + 0.01 * rng.standard_normal(t.size)).astype(np.float32)
    out = pred.speaker_diarization(a, sample_rate=16000, speaker_num=2)
    assert len(out) >= 1 and all(o['end'] > o['start'] for o in out)


def _wav(path, x):
    with wave.open(str(path), 'wb') as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000)
        w.writeframes(np.clip(x * 32767, -32768, 32767).astype('<i2').tobytes())


def test_evaluate_and_extract_features(golden, dirs, tmp_path):
    from mvector.trainer import MVectorTrainer
    from oracle import models as om
    _, meta = golden
    rng = np.random.default_rng(4)
    lines = []
    for i in range(10):
        n = int(rng.uniform(0.5, 3.0) * 16000)
        p = tmp_path / f'u{i}.wav'
        _wav(p, 0.2 * np.sin(2 * np.pi * rng.uniform(100, 400) * np.arange(n) / 16000) + 0.02 * rng.standard_normal(n))
        lines.append(f'{p}\t{i % 3}\n')
    lst = tmp_path / 'list.txt'
    lst.write_text(''.join(lines))
    cfg = _cfg(dirs['small_group'], meta['margs'], min_duration=0.3)
    cfg['dataset_conf'].update(train_list=str(lst), enroll_list=str(lst), trials_list=str(lst))
    tr = MVectorTrainer(cfg, use_gpu=True)
    tr._setup_eval()
    tr.model.load_state_dict(om.random_state_dict('EcapaTdnn', 32, seed=5, **meta['margs']))
    tr.model.eval()
    got, labels = tr._embed_list(str(lst))
    entries = tr._eval_order(str(lst))
    ref = []
    for s in range(0, len(entries), 4):
        items = [tr._eval_feature(p) for p, _ in entries[s:s + 4]]
        ref.append(tr.model(tr._zero_pad_features(items)).cpu().numpy())
    assert np.array_equal(got, np.concatenate(ref))
    eer, min_dcf, thr = tr.evaluate()
    assert np.isfinite(eer) and np.isfinite(min_dcf)
    out = tmp_path / 'feats'
    tr.extract_features(save_dir=str(out), max_duration=100)
    npys = sorted(str(p) for p in out.rglob('*.npy'))
    assert len(npys) >= 10
