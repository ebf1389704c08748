"""Write Hugging Face-style wav2vec 2.0 / WavLM checkpoint directories for the HF front-end tests: config.json,
preprocessor_config.json and the feature encoder's weights (seeded numpy default_rng) as model.safetensors, a sharded
model.safetensors.index.json or pytorch_model.bin.  Only the tensors `extract_features` depends on are written; the
transformer encoder's are not (the front-end never reads them, the reference initialises them at random)."""
import json
import os
import struct

import numpy as np

BASE = dict(conv_dim=(512,) * 7, conv_kernel=(10, 3, 3, 3, 3, 2, 2), conv_stride=(5, 2, 2, 2, 2, 2, 2))


def seeded_waves(B, L, seed, ratio=None):
    """[B, L] float32 noise at about 0.1 rms, the same bits on every machine: splitmix64 of the sample index and
    `seed` (integer arithmetic), three 24-bit uniforms summed exactly in float64, scaled and rounded once to float32.
    Row b is zero past round(ratio[b] * L), as predict_batch stages a ragged batch."""
    i = np.arange(3 * B * L, dtype=np.uint64)
    z = i + np.uint64(seed * 0x9E3779B97F4A7C15 % 2 ** 64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    u = (z >> np.uint64(40)).astype(np.float64) / 2.0 ** 24 - 0.5          # exact: 24-bit integers over 2^24
    w = ((u[0::3] + u[1::3] + u[2::3]) * 0.2).astype(np.float32).reshape(B, L)
    if ratio is not None:
        for b, r in enumerate(ratio):
            w[b, int(round(float(r) * L)):] = 0.0
    return w


def feature_weights(conv_dim, conv_kernel, norm, conv_bias, seed):
    """{name: float32 array} of the conv feature encoder and the projection LayerNorm (no prefix)."""
    rng = np.random.default_rng(seed)
    sd = {}
    cin = 1
    for i, (c, k) in enumerate(zip(conv_dim, conv_kernel)):
        p = f'feature_extractor.conv_layers.{i}.'
        sd[p + 'conv.weight'] = (rng.standard_normal((c, cin, k)) * np.sqrt(2.0 / (cin * k))).astype(np.float32)
        if conv_bias:
            sd[p + 'conv.bias'] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        if norm == 'layer' or i == 0:
            sd[p + 'layer_norm.weight'] = (1.0 + rng.standard_normal(c) * 0.1).astype(np.float32)
            sd[p + 'layer_norm.bias'] = (rng.standard_normal(c) * 0.1).astype(np.float32)
        cin = c
    sd['feature_projection.layer_norm.weight'] = (1.0 + rng.standard_normal(cin) * 0.1).astype(np.float32)
    sd['feature_projection.layer_norm.bias'] = (rng.standard_normal(cin) * 0.1).astype(np.float32)
    return sd


def write_safetensors(path, tensors, dtype='F32'):
    """numpy writer of the safetensors format: u64 header length, JSON header, raw little-endian tensors."""
    header, blobs, off = {}, [], 0
    for k, v in tensors.items():
        if dtype == 'F16':
            raw = v.astype(np.float16).tobytes()
        elif dtype == 'BF16':
            raw = (v.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16).tobytes()   # truncation: exact below
        else:
            raw = v.astype(np.float32).tobytes()
        header[k] = {'dtype': dtype, 'shape': list(v.shape), 'data_offsets': [off, off + len(raw)]}
        blobs.append(raw)
        off += len(raw)
    h = json.dumps(header).encode()
    h += b' ' * (-len(h) % 8)
    with open(path, 'wb') as f:
        f.write(struct.pack('<Q', len(h)))
        f.write(h)
        for b in blobs:
            f.write(b)


def write_hf_dir(d, model_type='wav2vec2', norm='group', conv_dim=(32,) * 7, conv_kernel=BASE['conv_kernel'],
                 conv_stride=BASE['conv_stride'], conv_bias=False, do_normalize=True, seed=0, fmt='safetensors',
                 prefix='', sampling_rate=16000, activation='gelu', dtype='F32', layer_norm_eps=1e-5, drop=()):
    """Write one checkpoint directory; returns the weights written (float32, unprefixed).  fmt: 'safetensors',
    'sharded' (two shards + index) or 'bin'; `drop`: tensor names left out."""
    os.makedirs(d, exist_ok=True)
    cfg = dict(model_type=model_type, architectures=['WavLMModel' if model_type == 'wavlm' else 'Wav2Vec2Model'],
               feat_extract_norm=norm, feat_extract_activation=activation, conv_dim=list(conv_dim),
               conv_kernel=list(conv_kernel), conv_stride=list(conv_stride), conv_bias=conv_bias,
               layer_norm_eps=layer_norm_eps, hidden_size=32, num_hidden_layers=1, num_attention_heads=2,
               intermediate_size=64, num_conv_pos_embeddings=16, num_conv_pos_embedding_groups=2,
               num_feat_extract_layers=len(conv_dim), do_stable_layer_norm=(norm == 'layer'))
    with open(os.path.join(d, 'config.json'), 'w') as f:
        json.dump(cfg, f, indent=1)
    pp = dict(feature_extractor_type='Wav2Vec2FeatureExtractor', feature_size=1, padding_side='right',
              padding_value=0.0, do_normalize=do_normalize, return_attention_mask=(norm == 'layer'),
              sampling_rate=sampling_rate)
    with open(os.path.join(d, 'preprocessor_config.json'), 'w') as f:
        json.dump(pp, f, indent=1)
    sd = feature_weights(conv_dim, conv_kernel, norm, conv_bias, seed)
    out = {prefix + k: v for k, v in sd.items() if k not in drop}
    if fmt == 'safetensors':
        write_safetensors(os.path.join(d, 'model.safetensors'), out, dtype)
    elif fmt == 'sharded':
        keys = list(out)
        shards = {'model-00001-of-00002.safetensors': keys[::2], 'model-00002-of-00002.safetensors': keys[1::2]}
        wmap = {}
        for name, ks in shards.items():
            write_safetensors(os.path.join(d, name), {k: out[k] for k in ks}, dtype)
            wmap.update({k: name for k in ks})
        with open(os.path.join(d, 'model.safetensors.index.json'), 'w') as f:
            json.dump({'metadata': {}, 'weight_map': wmap}, f)
    elif fmt == 'bin':
        import torch
        torch.save({k: torch.from_numpy(v) for k, v in out.items()}, os.path.join(d, 'pytorch_model.bin'))
    else:
        raise ValueError(fmt)
    return sd
