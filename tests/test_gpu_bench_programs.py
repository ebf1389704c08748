"""Every op of the programs bench.py times (c2-c5), at the bench batch and length, on the GPU's own inputs and held to
its engine's error bound (tests/bench_sweep.py).

The op tables (tests/op_cases.py) reach each kernel instance at up to 8 tiles per CTA and views under 1 GB; the bench
programs run up to 605 tiles per CTA, view offsets past 13 GB and up to 50 fp16-split amax slots.  Here each program
is run as its prefixes, one per op, on seeded waveforms through the product front-end (c5: the ragged batch with item
0 pinned to 10 s, T = 998, zero-masked tails), and every op is compared with the fp64 reference of that op on the
GPU's own fp32 operands: the tensor-core convs on one M tile of every CTA index and every tile ordinal (first, last and
a seeded row) and on every row of the first and the last utterance, the other kernels on their first and last rows,
their grid-stride wraps and a seeded sample, the pooling ops and small-M linears on every row.  Copies and max pooling
must be bit-exact, and every output finite where the reference is."""
import os
import time

import numpy as np
import pytest
import torch

import bench_sweep as bs
import op_cases as oc

pytestmark = pytest.mark.gpu


def _features(cfg, name):
    """Features [B, T, F] of the bench batch: bench.batch_lens / synth_waves through the product front-end."""
    import bench
    from mvector.data_utils.featurizer import AudioFeaturizer
    B = cfg['per_gpu']
    lens = bench.batch_lens(cfg, B, 1234 + cfg['idx'])
    if cfg['ragged']:
        lens[0] = 160000                                   # T = 998, as test_gpu_baseline_sizes pins it
    lmax = max(lens)
    x = torch.zeros(B, lmax)
    for j, w in enumerate(bench.synth_waves(lens, 1234 + 1000 * cfg['idx'])):
        x[j, :w.shape[0]] = torch.from_numpy(w)
    fz = AudioFeaturizer(feature_method=cfg['feature'], method_args=dict(cfg['fargs']))
    T = fz.num_frames(lmax)
    assert T == oc.BENCH_T[name], (name, T)
    keep = None
    if cfg['ragged']:
        keep = fz.keep_frames(torch.tensor([n / lmax for n in lens], dtype=torch.float32), T).cuda()
    feats = fz.forward_keep(x.cuda().contiguous(), keep)
    torch.cuda.synchronize()
    return feats


@pytest.mark.parametrize('name', ['c2', 'c3', 'c4', 'c5'])
def test_bench_program_op_by_op(name):
    model, cfg = oc.bench_model(name)
    feats = _features(cfg, name)
    pb = model.lower(cfg['per_gpu'], oc.BENCH_T[name]).finalize()
    engines = [oc.engine_of(o) for o in pb.ops]
    t0 = time.time()
    sw = bs.Sweep(name, pb, model._blob, engines, bs.GpuBackend(model._blob, feats))
    stats = sw.run(workers=min(8, os.cpu_count() or 1),
                   log=lambda i: i % 10 or print(f'{name}: op {i} at {time.time() - t0:.0f} s', flush=True))   # run, then checked
    print(f'\n{name}: {len(pb.ops)} ops checked in {time.time() - t0:.0f} s')
    for k, (r, n) in sorted(stats.items()):
        print(f'  {name} {k:20s} worst err/beta {r:.3f} over {n} elements')
    assert sum(1 for _ in sw.ops) == len(pb.ops)
    assert all(r <= 1.0 for r, _ in stats.values())
