"""Generate tests/golden/hf_frontend.npz by running the UNMODIFIED reference (/root/reference) with transformers:

    python tests/golden/make_hf_golden.py

Each case writes an HF checkpoint directory with tests/hf_writer.py (seeded, so the GPU tests rebuild the same
directory without this script, the reference or transformers), runs the reference
AudioFeaturizer(feature_method=<dir>, use_hf_model=True) on CPU and a reference EcapaTdnn(input_size=conv_dim[-1])
with seeded weights (oracle.models.random_state_dict) on those features, and stores the inputs, features and
embeddings.  The waveforms are not stored: tests/hf_writer.py::seeded_waves rebuilds them bit for bit from the seed in
the file's metadata.  Of the features every `feat_step`-th channel is stored (16 per case), which keeps the file small;
the embeddings come from the full features.  The transformers version used is recorded in the file.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = '/root/reference'
sys.path.insert(0, REF)
sys.path.insert(1, ROOT)
sys.path.insert(2, os.path.join(ROOT, 'tests'))

MARGS = dict(embd_dim=32, pooling_type='ASP', channels=[64, 64, 64, 64, 192])

# name: (writer kwargs, B, L, lens_ratio)
CASES = {
    'small_group': (dict(model_type='wav2vec2', norm='group', conv_dim=(32,) * 7, seed=1), 3, 16000, [1.0, 0.75, 0.5]),
    'small_group_raw': (dict(model_type='wav2vec2', norm='group', conv_dim=(48,) * 7, do_normalize=False, seed=2), 2,
                        12000, [1.0, 0.6]),
    'small_layer': (dict(model_type='wavlm', norm='layer', conv_dim=(48,) * 7, conv_bias=True, seed=3), 3, 16000,
                    [0.8, 1.0, 0.55]),
    'small_layer_raw': (dict(model_type='wavlm', norm='layer', conv_dim=(64,) * 7, conv_bias=True, do_normalize=False,
                             seed=4), 2, 9000, [1.0, 0.9]),
    'base_1s': (dict(model_type='wav2vec2', norm='group', conv_dim=(512,) * 7, seed=5), 2, 16000, [1.0, 0.7]),
    'base_3s': (dict(model_type='wav2vec2', norm='group', conv_dim=(512,) * 7, seed=6), 2, 48000, [1.0, 0.4]),
}


def main():
    import transformers
    from hf_writer import seeded_waves, write_hf_dir
    from mvector.data_utils.featurizer import AudioFeaturizer
    from mvector.models.ecapa_tdnn import EcapaTdnn
    from oracle.models import random_state_dict

    out, meta = {}, {'transformers': transformers.__version__, 'torch': torch.__version__, 'np': np.__version__,
                     'margs': MARGS, 'cases': {}}
    for ci, (name, (kw, B, L, ratio)) in enumerate(CASES.items()):
        wave = seeded_waves(B, L, 100 + ci, ratio)
        with tempfile.TemporaryDirectory() as td:
            write_hf_dir(td, **kw)
            fz = AudioFeaturizer(feature_method=td, use_hf_model=True, method_args={'use_gpu': False})
            feats = fz(torch.from_numpy(wave), torch.tensor(ratio, dtype=torch.float32))
        F = feats.shape[2]
        sd = random_state_dict('EcapaTdnn', F, seed=ci, **MARGS)
        m = EcapaTdnn(input_size=F, **MARGS)
        m.load_state_dict(sd)
        m.eval()
        with torch.no_grad():
            emb = m(feats)
        step = F // 16
        out[name + '/feats'] = np.ascontiguousarray(feats.numpy()[:, :, ::step], dtype=np.float32)
        out[name + '/emb'] = emb.numpy().astype(np.float32)
        meta['cases'][name] = dict(writer={k: (list(v) if isinstance(v, tuple) else v) for k, v in kw.items()},
                                   model_seed=ci, B=B, L=L, wave_seed=100 + ci, ratio=ratio, feat_step=step)
        print(name, tuple(feats.shape), tuple(emb.shape))
    out['meta'] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(os.path.join(HERE, 'hf_frontend.npz'), **out)


if __name__ == '__main__':
    main()
