"""Hugging Face wav2vec 2.0 / WavLM checkpoints for the HF front-end, read without `transformers` and never downloaded.

The reference passes `feature_method` to `AutoFeatureExtractor.from_pretrained` / `AutoModel.from_pretrained`
(featurizer.py:31-33) and keeps only `outputs.extract_features`, which depend on the processor's normalisation and the
model's convolutional feature encoder plus the feature projection's LayerNorm.  This module resolves the same name to a
local directory (the directory itself, or a hub id already in the local Hugging Face cache) and reads exactly what
those need from `config.json`, `preprocessor_config.json` and the weights.
"""
import json
import os
import struct

import numpy as np

# Wav2Vec2Config / WavLMConfig defaults of the fields the feature encoder uses
_CONFIG_DEFAULTS = dict(feat_extract_norm='group', feat_extract_activation='gelu', conv_dim=(512,) * 7,
                        conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_stride=(5, 2, 2, 2, 2, 2, 2), conv_bias=False,
                        layer_norm_eps=1e-5)
_MODEL_TYPES = ('wav2vec2', 'wavlm')
_PREFIXES = ('', 'wav2vec2.', 'wavlm.')
_ST_DTYPES = {'F32': np.float32, 'F64': np.float64, 'F16': np.float16, 'BF16': None}


class HfModelNotLocal(OSError, NotImplementedError):
    """`feature_method` names no local checkpoint.  An OSError, as `from_pretrained` raises for a model it cannot
    find, and a NotImplementedError, as for every option this path does not run: downloading is deliberately not
    implemented."""


def cache_dirs():
    """The hub caches searched for a model id, in the order huggingface_hub resolves them."""
    out = []
    if os.environ.get('HF_HUB_CACHE'):
        out.append(os.environ['HF_HUB_CACHE'])
    if os.environ.get('HF_HOME'):
        out.append(os.path.join(os.environ['HF_HOME'], 'hub'))
    out.append(os.path.join(os.path.expanduser('~'), '.cache', 'huggingface', 'hub'))
    return list(dict.fromkeys(out))


def resolve(name):
    """`feature_method` -> the local directory holding the checkpoint: the directory itself, or the snapshot that
    refs/main of `models--{org}--{name}` points at in a local hub cache.  Never downloads: an id found nowhere raises
    HfModelNotLocal (an OSError) naming every place searched."""
    name = os.fspath(name)
    if os.path.isdir(name):
        return name
    searched = [os.path.abspath(name)]
    repo = 'models--' + name.replace('/', '--')
    for cache in cache_dirs():
        root = os.path.join(cache, repo)
        searched.append(root)
        ref = os.path.join(root, 'refs', 'main')
        if not os.path.isfile(ref):
            continue
        with open(ref) as f:
            snap = os.path.join(root, 'snapshots', f.read().strip())
        if os.path.isfile(os.path.join(snap, 'config.json')):
            return snap
    raise HfModelNotLocal(f'HF model {name!r} is neither a local directory nor in a local Hugging Face cache (it is '
                          f'never downloaded); searched: ' + ', '.join(searched))


def _bf16_to_f32(raw):
    return (np.frombuffer(raw, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def read_safetensors(path, wanted=None):
    """{name: float32 ndarray} of a .safetensors file (8-byte little-endian header length, JSON header, raw tensors).
    F16 / BF16 / F64 tensors are converted to float32.  `wanted`: names to read (default all)."""
    out = {}
    with open(path, 'rb') as f:
        (n,) = struct.unpack('<Q', f.read(8))
        header = json.loads(f.read(n))
        base = 8 + n
        for key, info in header.items():
            if key == '__metadata__' or (wanted is not None and key not in wanted):
                continue
            dt = info['dtype']
            if dt not in _ST_DTYPES:
                raise ValueError(f'{path}: tensor {key} has dtype {dt}; the HF front-end reads F32, F16, BF16 and F64')
            b, e = info['data_offsets']
            f.seek(base + b)
            raw = f.read(e - b)
            a = _bf16_to_f32(raw) if dt == 'BF16' else np.frombuffer(raw, dtype=_ST_DTYPES[dt])
            out[key] = np.ascontiguousarray(a.astype(np.float32).reshape(info['shape']))
    return out


def _read_bin(path):
    import torch
    sd = torch.load(path, map_location='cpu', weights_only=True)
    return {k: v.detach().to(torch.float32).numpy() for k, v in sd.items()}


def read_weights(d, wanted):
    """The tensors named in `wanted` (any of the accepted key prefixes) from model.safetensors, a sharded
    model.safetensors.index.json or pytorch_model.bin, whichever the directory has first."""
    cands = {p + k for p in _PREFIXES for k in wanted}
    st, idx, pt = (os.path.join(d, n) for n in ('model.safetensors', 'model.safetensors.index.json', 'pytorch_model.bin'))
    if os.path.isfile(st):
        return read_safetensors(st, cands)
    if os.path.isfile(idx):
        with open(idx) as f:
            wmap = json.load(f)['weight_map']
        out = {}
        for shard in sorted({wmap[k] for k in cands if k in wmap}):
            out.update(read_safetensors(os.path.join(d, shard), cands))
        return out
    if os.path.isfile(pt):
        return {k: v for k, v in _read_bin(pt).items() if k in cands}
    raise OSError(f'{d} has no model.safetensors, model.safetensors.index.json or pytorch_model.bin')


class HfCheckpoint:
    """What the HF front-end needs of a checkpoint: the conv stack geometry, the norms, the processor's normalisation
    and the weights (float32), named as in Wav2Vec2Model / WavLMModel without prefix."""

    def __init__(self, name):
        self.path = resolve(name)
        with open(os.path.join(self.path, 'config.json')) as f:
            cfg = json.load(f)
        mt = cfg.get('model_type')
        if mt not in _MODEL_TYPES:
            raise NotImplementedError(f'model_type {mt!r}: the HF front-end runs wav2vec2 and wavlm checkpoints '
                                      '(their extract_features)')
        self.model_type = mt
        c = dict(_CONFIG_DEFAULTS)
        c.update({k: cfg[k] for k in _CONFIG_DEFAULTS if k in cfg})
        if c['feat_extract_activation'] != 'gelu':
            raise NotImplementedError(f"feat_extract_activation {c['feat_extract_activation']!r}: the HF front-end "
                                      "runs 'gelu'")
        if c['feat_extract_norm'] not in ('group', 'layer'):
            raise ValueError(f"`config.feat_extract_norm` is {c['feat_extract_norm']}, but has to be one of ['group', "
                             "'layer']")
        self.norm = c['feat_extract_norm']
        self.conv_dim = [int(v) for v in c['conv_dim']]
        self.conv_kernel = [int(v) for v in c['conv_kernel']]
        self.conv_stride = [int(v) for v in c['conv_stride']]
        if not (len(self.conv_dim) == len(self.conv_kernel) == len(self.conv_stride)):
            raise ValueError('Configuration for convolutional layers is incorrect: conv_dim, conv_stride and conv_kernel '
                             'must have the same length')
        self.conv_bias = bool(c['conv_bias'])
        self.layer_norm_eps = float(c['layer_norm_eps'])
        pp = {}
        ppath = os.path.join(self.path, 'preprocessor_config.json')
        if os.path.isfile(ppath):
            with open(ppath) as f:
                pp = json.load(f)
        self.do_normalize = bool(pp.get('do_normalize', True))
        self.sampling_rate = int(pp.get('sampling_rate', 16000))
        if self.sampling_rate != 16000:
            raise ValueError(f'The model corresponding to this feature extractor was trained using a sampling_rate of '
                             f'{self.sampling_rate}. Please make sure that the provided `raw_speech` input was sampled '
                             f'with {self.sampling_rate} and not 16000.')
        need = self.tensor_names()
        found = read_weights(self.path, need)
        self.weights, missing = {}, []
        for k in need:
            hit = [p + k for p in _PREFIXES if p + k in found]
            if hit:
                self.weights[k] = found[hit[0]]
            else:
                missing.append(k)
        if missing:
            raise RuntimeError(f'Error(s) in loading state_dict for {type(self).__name__}:\n\tMissing key(s) in '
                               'state_dict: ' + ', '.join(f'"{k}"' for k in missing) + f' ({self.path})')

    def tensor_names(self):
        n = []
        for i in range(len(self.conv_dim)):
            p = f'feature_extractor.conv_layers.{i}.'
            n.append(p + 'conv.weight')
            if self.conv_bias:
                n.append(p + 'conv.bias')
            if self.norm == 'layer' or i == 0:
                n += [p + 'layer_norm.weight', p + 'layer_norm.bias']
        return n + ['feature_projection.layer_norm.weight', 'feature_projection.layer_norm.bias']

    def num_frames(self, n):
        """Frames of an n-sample waveform through the conv stack (0 when too short)."""
        t = int(n)
        for k, s in zip(self.conv_kernel, self.conv_stride):
            t = 0 if t < k else (t - k) // s + 1
        return t

    @property
    def feature_dim(self):
        return self.conv_dim[-1]
