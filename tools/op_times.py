"""Per-op device times of the ECAPA B=256 program (dev tool): the mean time of each tensor-core conv class
(engine, M x N x K) over three profiled runs."""
import json, sys, collections
sys.path.insert(0, '.')
import torch
import __graft_entry__ as ge
ge.build()
from mvector.models import build_model
from mvector.utils.utils import dict_to_object
from oracle import models as om
from loguru import logger
logger.remove()
margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
m = build_model(80, dict_to_object({'model_conf': {'model': 'EcapaTdnn', 'model_args': margs}}))
m.load_state_dict(om.random_state_dict('EcapaTdnn', 80, seed=0, **margs))
B, T = 256, 298
prog = m.program(B, T)
f = torch.randn(B, T, 80, device='cuda')
e = torch.empty(B, 192, device='cuda')
for _ in range(2): prog.run(f, e)
acc = None
for _ in range(3):
    ops = prog.run_profiled(f, e)
    if acc is None: acc = ops
    else:
        for a, o in zip(acc, ops): a['ms'] += o['ms']
agg = collections.OrderedDict()
for o in acc:
    key = (o['kind'], o['engine'], o['M'], o['N'], o['K'])
    a = agg.setdefault(key, [0, 0.0]); a[0] += 1; a[1] += o['ms'] / 3
tot = sum(v[1] for v in agg.values())
# a fused Res2Net chain books its launch on the chain's first op and ~0 on the rest (vp_embed_profiled)
chain = [o['ms'] for o in acc if o['kind'] == 1 and o['engine'] == 2 and o['N'] <= 64 and o['K'] == 3 * o['N']]
if chain:
    print('res2 chain convs (N <= 64, k3): %d ops, %.3f ms in all' % (len(chain), sum(chain) / 3))
print('total %.3f ms' % tot, ' | '.join(f"{'tf32' if k[1] == 2 else 'fp16'} {k[2]}x{k[3]}x{k[4]}:{v[1]/v[0]:.3f}"
                                        for k, v in agg.items() if k[0] == 1 and k[1] in (2, 3)))
