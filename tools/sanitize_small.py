"""Tiny workload for compute-sanitizer (memcheck / racecheck): small-config ECAPA + CAM++ from waveforms, a small
fused Res2Net chain and a small HF wav2vec 2.0 / WavLM front-end."""
import sys
sys.path.insert(0, '.'); sys.path.insert(0, 'tests')
import json, numpy as np, torch
from loguru import logger
logger.remove()
from conftest import load_golden
from mvector.models import build_model
from mvector.utils.utils import dict_to_object
from mvector.data_utils.featurizer import AudioFeaturizer
man = json.load(open('tests/golden/manifest.json'))
for name in ('ecapa_small', 'campplus_small', 'eres2net_small'):
    m = man[name]
    z, sd = load_golden(name)
    model = build_model(m['feature_dim'], dict_to_object({'model_conf': {'model': m['model'], 'model_args': m['model_args']}}))
    model.load_state_dict(sd)
    fz = AudioFeaturizer(m['preprocess']['feature_method'], method_args=m['preprocess']['method_args'])
    w = np.stack([z['wave0'][:7360], z['wave1'][:7360]])
    emb = model(fz(torch.from_numpy(w))).cpu().numpy()
    # big enough M for the tensor-core engine too
    feats = torch.from_numpy(np.tile(z['feats'][:1], (24, 1, 1))).cuda()
    emb2 = model(feats).cpu().numpy()
    print(name, emb.shape, float(np.abs(emb).max()), emb2.shape, flush=True)
# a small fused Res2Net chain (res2_chain_kernel): its last row block reads past the plane chunks it uses, and it
# rewrites its planes in place between convs; once with y untracked, once with an amax slot
import test_gpu_res2_chain as r2
for tracked in (False, True):
    fused, ref, launches, _, slot = r2._run(8, 130, 32, 2, 3, tracked=tracked)
    print('res2 chain', 'tracked' if tracked else 'untracked', launches, slot, flush=True)
# a small HF wav2vec 2.0 front-end (hf.cu), padded and ragged, both norms
import tempfile
from hf_writer import write_hf_dir
for norm in ('group', 'layer'):
    with tempfile.TemporaryDirectory() as td:
        write_hf_dir(td, model_type='wav2vec2' if norm == 'group' else 'wavlm', norm=norm, conv_dim=(32,) * 7,
                     conv_bias=norm == 'layer', seed=1)
        fz = AudioFeaturizer(td, use_hf_model=True)
        w = torch.randn(3, 4001, device='cuda') * 0.1
        f = fz(w, torch.tensor([1.0, 0.5, 0.8]))
        fe, tb = fz.forward_each(w, [4001, 400, 2999])
        print('hf', norm, tuple(f.shape), tuple(fe.shape), tb.tolist(), flush=True)
print('done')
