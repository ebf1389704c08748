"""CPU restatement of the reference's HF front-end (featurizer.py:65-90 with a wav2vec 2.0 / WavLM checkpoint), from
the weights alone: Wav2Vec2FeatureExtractor's numpy float32 normalisation, the conv feature encoder, the feature
projection's LayerNorm (its `extract_features`), then CMN and the lens_ratio mask -- the same torch fp32 CPU ops the
reference runs, so its result equals the reference's bit for bit."""
import numpy as np
import torch
import torch.nn.functional as F


def processor_normalize(w):
    """zero_mean_unit_var_norm of Wav2Vec2FeatureExtractor on one float32 row."""
    w = np.asarray(w, dtype=np.float32)
    return (w - w.mean()) / np.sqrt(w.var() + 1e-7)


def extract_features(waves, sd, norm, conv_kernel, conv_stride, do_normalize=True, layer_norm_eps=1e-5,
                     dtype=torch.float32):
    """waves [B, L] float32 -> extract_features [B, T, C] (torch float32; dtype=torch.float64 evaluates the same
    formula in fp64 from the processor's float32 output on, the exact value the fp32 computations round)."""
    w = np.asarray(waves, dtype=np.float32)
    if do_normalize:
        w = np.stack([processor_normalize(r) for r in w])
    h = torch.from_numpy(np.ascontiguousarray(w))[:, None, :].to(dtype)
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)
    for i, (k, s) in enumerate(zip(conv_kernel, conv_stride)):
        p = f'feature_extractor.conv_layers.{i}.'
        h = F.conv1d(h, t(sd[p + 'conv.weight']), t(sd[p + 'conv.bias']) if p + 'conv.bias' in sd else None, stride=s)
        if norm == 'group' and i == 0:
            h = F.group_norm(h, h.shape[1], t(sd[p + 'layer_norm.weight']), t(sd[p + 'layer_norm.bias']), eps=1e-5)
        elif norm == 'layer':
            h = F.layer_norm(h.transpose(1, 2), (h.shape[1],), t(sd[p + 'layer_norm.weight']),
                             t(sd[p + 'layer_norm.bias']), eps=1e-5).transpose(1, 2)
        h = F.gelu(h)
    h = h.transpose(1, 2)
    return F.layer_norm(h, (h.shape[2],), t(sd['feature_projection.layer_norm.weight']),
                        t(sd['feature_projection.layer_norm.bias']), eps=layer_norm_eps)


def featurize(waves, ratio, sd, norm, conv_kernel, conv_stride, do_normalize=True, layer_norm_eps=1e-5,
              dtype=torch.float32):
    """The reference AudioFeaturizer.forward with use_hf_model: extract_features, CMN, lens_ratio mask."""
    f = extract_features(waves, sd, norm, conv_kernel, conv_stride, do_normalize, layer_norm_eps, dtype)
    f = f - f.mean(1, keepdim=True)
    if ratio is not None:
        T = f.shape[1]
        keep = torch.round(torch.as_tensor(ratio, dtype=torch.float32) * T).long()
        f = torch.where(torch.arange(T)[None, :, None] < keep[:, None, None], f, torch.zeros_like(f))
    return f
