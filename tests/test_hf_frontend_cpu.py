"""HF wav2vec 2.0 / WavLM front-end, host side (no GPU): the CPU restatement against the reference's golden features,
checkpoint loading (key prefixes, safetensors / sharded index / .bin, half-precision upcast, hub-cache resolution),
every refusal, and the frame counts of the conv stack."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT

sys.path.insert(0, os.path.join(ROOT, 'tests'))
from hf_writer import feature_weights, write_hf_dir  # noqa: E402
import hf_oracle  # noqa: E402

REF = '/root/reference'


def _golden():
    z = np.load(os.path.join(GOLDEN, 'hf_frontend.npz'))
    return z, json.loads(bytes(z['meta']).decode())


def _writer_kw(meta, name):
    kw = dict(meta['cases'][name]['writer'])
    for k in ('conv_dim', 'conv_kernel', 'conv_stride'):
        if k in kw:
            kw[k] = tuple(kw[k])
    return kw


def _waves(meta, name):
    from hf_writer import seeded_waves
    c = meta['cases'][name]
    return seeded_waves(c['B'], c['L'], c['wave_seed'], c['ratio']), np.asarray(c['ratio'], np.float32)


def _oracle_feats(meta, name):
    kw = _writer_kw(meta, name)
    sd = feature_weights(kw['conv_dim'], (10, 3, 3, 3, 3, 2, 2), kw['norm'], kw.get('conv_bias', False), kw['seed'])
    wave, ratio = _waves(meta, name)
    return hf_oracle.featurize(wave, ratio, sd, kw['norm'], (10, 3, 3, 3, 3, 2, 2), (5, 2, 2, 2, 2, 2, 2),
                               kw.get('do_normalize', True))


@pytest.mark.parametrize('name', ['small_group', 'small_group_raw', 'small_layer', 'small_layer_raw', 'base_1s',
                                  'base_3s'])
def test_oracle_matches_reference_golden(name):
    """The restatement reproduces the reference's features (produced with transformers, recorded in the file; every
    feat_step-th channel stored)."""
    z, meta = _golden()
    got = _oracle_feats(meta, name).numpy()[:, :, ::meta['cases'][name]['feat_step']]
    want = z[name + '/feats']
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= 1e-5


def test_seeded_waves_are_fixed():
    """The golden's inputs are rebuilt from integer arithmetic: pin a few of their bits."""
    from hf_writer import seeded_waves
    w = seeded_waves(2, 1000, 7, [1.0, 0.5])
    assert w.dtype == np.float32 and (w[1, 500:] == 0).all() and 0.08 < float(w[0].std()) < 0.12
    assert w.view(np.uint32)[0, :4].tolist() == [1029923498, 1037942984, 1018949670, 1004329523]


def _reference_available():
    try:
        import transformers  # noqa: F401
    except ImportError:
        return False
    return os.path.isdir(os.path.join(REF, 'mvector'))


@pytest.mark.skipif(not _reference_available(), reason='needs the reference tree and transformers')
@pytest.mark.parametrize('norm,model_type', [('group', 'wav2vec2'), ('layer', 'wavlm')])
def test_oracle_equals_live_reference(tmp_path, norm, model_type):
    """Bit for bit against the reference's AudioFeaturizer(use_hf_model=True) on the same machine."""
    import subprocess
    d = str(tmp_path / 'm')
    sd = write_hf_dir(d, model_type=model_type, norm=norm, conv_dim=(32,) * 7, conv_bias=norm == 'layer', seed=7)
    rng = np.random.default_rng(3)
    wave = (rng.standard_normal((3, 8000)) * 0.1).astype(np.float32)
    wave[1, 5000:] = 0
    ratio = np.array([1.0, 0.625, 1.0], np.float32)
    np.save(tmp_path / 'w.npy', wave)
    np.save(tmp_path / 'r.npy', ratio)
    code = ('import sys, numpy as np, torch; sys.path.insert(0, %r)\n'
            'from mvector.data_utils.featurizer import AudioFeaturizer\n'
            'af = AudioFeaturizer(feature_method=%r, use_hf_model=True, method_args={"use_gpu": False})\n'
            'f = af(torch.from_numpy(np.load(%r)), torch.from_numpy(np.load(%r)))\n'
            'np.save(%r, f.numpy())\n') % (REF, d, str(tmp_path / 'w.npy'), str(tmp_path / 'r.npy'),
                                           str(tmp_path / 'f.npy'))
    subprocess.run([sys.executable, '-c', code], check=True, capture_output=True, cwd=str(tmp_path))
    ref = np.load(tmp_path / 'f.npy')
    got = hf_oracle.featurize(wave, ratio, sd, norm, (10, 3, 3, 3, 3, 2, 2), (5, 2, 2, 2, 2, 2, 2)).numpy()
    assert np.array_equal(got, ref)


# ------------------------------------------------------------------------------------------------ loading
def _load(d):
    from mvector.data_utils.hf_checkpoint import HfCheckpoint
    return HfCheckpoint(d)


@pytest.mark.parametrize('fmt', ['safetensors', 'sharded', 'bin'])
@pytest.mark.parametrize('prefix', ['', 'wav2vec2.', 'wavlm.'])
def test_loader_formats_and_prefixes(tmp_path, fmt, prefix):
    sd = write_hf_dir(str(tmp_path), norm='layer', conv_dim=(16, 24, 32, 16, 16, 16, 20), conv_bias=True, seed=11,
                      fmt=fmt, prefix=prefix)
    c = _load(str(tmp_path))
    assert c.norm == 'layer' and c.conv_bias and c.feature_dim == 20 and c.do_normalize
    assert sorted(c.weights) == sorted(sd)
    for k, v in sd.items():
        assert c.weights[k].dtype == np.float32 and np.array_equal(c.weights[k], v), k


@pytest.mark.parametrize('dtype', ['F16', 'BF16'])
def test_loader_upcasts_half_precision(tmp_path, dtype):
    sd = write_hf_dir(str(tmp_path), conv_dim=(16,) * 7, seed=12, dtype=dtype)
    c = _load(str(tmp_path))
    for k, v in sd.items():
        if dtype == 'F16':
            want = v.astype(np.float16).astype(np.float32)
        else:
            want = (v.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)
        assert c.weights[k].dtype == np.float32 and np.array_equal(c.weights[k], want), k


def _fake_cache(root, repo_id, tmp_src):
    d = os.path.join(root, 'models--' + repo_id.replace('/', '--'))
    os.makedirs(os.path.join(d, 'refs'))
    with open(os.path.join(d, 'refs', 'main'), 'w') as f:
        f.write('abc123')
    snap = os.path.join(d, 'snapshots', 'abc123')
    os.makedirs(os.path.dirname(snap))
    os.rename(tmp_src, snap)
    return snap


@pytest.mark.parametrize('var', ['HF_HUB_CACHE', 'HF_HOME'])
def test_hub_id_resolves_from_local_cache(tmp_path, monkeypatch, var):
    from mvector.data_utils.hf_checkpoint import resolve
    src = str(tmp_path / 'src')
    write_hf_dir(src, conv_dim=(16,) * 7, seed=13)
    cache = str(tmp_path / 'cache')
    snap = _fake_cache(cache if var == 'HF_HUB_CACHE' else os.path.join(cache, 'hub'), 'acme/tiny-w2v', src)
    monkeypatch.delenv('HF_HUB_CACHE', raising=False)
    monkeypatch.delenv('HF_HOME', raising=False)
    monkeypatch.setenv(var, cache)
    assert resolve('acme/tiny-w2v') == snap
    assert _load('acme/tiny-w2v').feature_dim == 16


def test_uncached_hub_id_names_the_places_searched(tmp_path, monkeypatch):
    monkeypatch.setenv('HF_HUB_CACHE', str(tmp_path / 'c1'))
    monkeypatch.setenv('HF_HOME', str(tmp_path / 'h'))
    with pytest.raises(OSError) as e:
        _load('facebook/wav2vec2-base')
    msg = str(e.value)
    assert 'never' in msg and 'facebook/wav2vec2-base' in msg
    assert os.path.join(str(tmp_path / 'c1'), 'models--facebook--wav2vec2-base') in msg
    assert os.path.join(str(tmp_path / 'h'), 'hub', 'models--facebook--wav2vec2-base') in msg


# ------------------------------------------------------------------------------------------------ refusals
def _edit_json(path, **kv):
    with open(path) as f:
        j = json.load(f)
    j.update(kv)
    with open(path, 'w') as f:
        json.dump(j, f)


def test_refusals_name_the_field(tmp_path):
    d = str(tmp_path)
    write_hf_dir(d, conv_dim=(16,) * 7, seed=14)
    _edit_json(os.path.join(d, 'config.json'), model_type='hubert')
    with pytest.raises(NotImplementedError, match='hubert'):
        _load(d)
    _edit_json(os.path.join(d, 'config.json'), model_type='wav2vec2', feat_extract_activation='relu')
    with pytest.raises(NotImplementedError, match='feat_extract_activation.*relu'):
        _load(d)
    _edit_json(os.path.join(d, 'config.json'), feat_extract_activation='gelu', feat_extract_norm='batch')
    with pytest.raises(ValueError, match='feat_extract_norm'):
        _load(d)
    _edit_json(os.path.join(d, 'config.json'), feat_extract_norm='group')
    _edit_json(os.path.join(d, 'preprocessor_config.json'), sampling_rate=8000)
    with pytest.raises(ValueError, match='sampling_rate of 8000'):
        _load(d)
    _edit_json(os.path.join(d, 'preprocessor_config.json'), sampling_rate=16000)
    assert _load(d).feature_dim == 16


def test_missing_tensor_is_refused_by_name(tmp_path):
    d = str(tmp_path)
    write_hf_dir(d, conv_dim=(16,) * 7, seed=15, drop=('feature_extractor.conv_layers.3.conv.weight',))
    with pytest.raises(RuntimeError, match=r'Missing key.*feature_extractor\.conv_layers\.3\.conv\.weight'):
        _load(d)
    d2 = str(tmp_path / 'b')
    write_hf_dir(d2, conv_dim=(16,) * 7, seed=15, drop=('feature_projection.layer_norm.bias',))
    with pytest.raises(RuntimeError, match='feature_projection.layer_norm.bias'):
        _load(d2)


# ------------------------------------------------------------------------------------------------ frames
def test_frame_counts_every_residue(tmp_path):
    """num_frames equals the conv stack's output length for every length residue mod 5 and mod 2 of each layer."""
    d = str(tmp_path)
    sd = write_hf_dir(d, conv_dim=(16,) * 7, seed=16)
    c = _load(d)
    for n in list(range(395, 480)) + [16000, 16001, 16004, 24321, 48000]:
        if n < 400:
            assert c.num_frames(n) == 0
            continue
        w = np.random.default_rng(n).standard_normal((1, n)).astype(np.float32)
        f = hf_oracle.extract_features(w, sd, 'group', c.conv_kernel, c.conv_stride)
        assert c.num_frames(n) == f.shape[1], n
    assert c.num_frames(400) == 1 and c.num_frames(399) == 0
    assert c.num_frames(24000) == 74                     # a 1.5 s diarization chunk


def test_featurizer_builds_without_gpu(tmp_path):
    from mvector.data_utils.featurizer import AudioFeaturizer
    d = str(tmp_path)
    write_hf_dir(d, model_type='wavlm', norm='layer', conv_dim=(16,) * 6 + (24,), conv_bias=True, seed=17)
    fz = AudioFeaturizer(feature_method=d, use_hf_model=True, method_args={'use_gpu': True})
    assert fz.feature_dim == 24 and fz.num_frames(16000) == 49 and not fz.whole_call
    with pytest.raises(OSError):
        AudioFeaturizer(feature_method=str(tmp_path / 'nope'), use_hf_model=True)
