"""Tiny workload for compute-sanitizer (memcheck / racecheck): small-config ECAPA + CAM++ from waveforms, and a small
fused Res2Net chain."""
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
print('done')
