"""Host-side timeline of MVectorPredictor.predict_batch (ECAPA c2: 256 x 3 s host arrays) + a sweep of the staging knobs.
Dev tool: prints where the end-to-end time goes; not a bench value."""
import json, os, sys, tempfile, time
sys.path.insert(0, '.')
import numpy as np
import torch
import __graft_entry__ as ge
ge.build()
from loguru import logger
logger.remove()
import bench
from mvector.predict import MVectorPredictor

cfg = bench.CONFIGS[sys.argv[1] if len(sys.argv) > 1 else 'c2']
td = tempfile.mkdtemp()
bench.save_weights(cfg, td)
pred = MVectorPredictor(configs=bench.yml_config(cfg), model_path=td, use_gpu=True)
B = cfg['per_gpu']
pools = [bench.synth_waves(bench.batch_lens(cfg, B, 10 + i), 20 + i) for i in range(4)]


def run(n, trace=False):
    ts = []
    for i in range(n):
        torch.cuda.synchronize()
        pred._trace = [] if trace else None
        pred._trace_dev = [] if trace else None
        t0 = time.perf_counter()
        pred.predict_batch(pools[i % 4])
        t1 = time.perf_counter()
        ts.append((t1 - t0) * 1e3)
        if trace and i == n - 1:
            prev = t0
            for label, t in pred._trace:
                print(f'    +{(t - prev) * 1e3:7.3f} ms  {label}')
                prev = t
            print(f'    +{(t1 - prev) * 1e3:7.3f} ms  return')
            torch.cuda.synchronize()
            e0 = pred._trace_dev[0][1]
            host0 = dict(pred._trace)['host prep done (keep, buffers, pointer table)']
            print(f'    device events, ms after the host-prep mark (which is {(host0 - t0) * 1e3:.3f} ms into the call):')
            for label, e in pred._trace_dev[1:]:
                print(f'      {e0.elapsed_time(e):7.3f}  {label}')
    pred._trace = None
    pred._trace_dev = None
    return ts


# PCIe ceiling of this box: one pinned -> device copy of the step's input bytes, device-timed
nbytes = sum(w.nbytes for w in pools[0])
hp = torch.empty(nbytes // 4, dtype=torch.float32).pin_memory()
dp = torch.empty(nbytes // 4, dtype=torch.float32, device='cuda')
for _ in range(3):
    dp.copy_(hp, non_blocking=True)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    dp.copy_(hp, non_blocking=True)
e1.record()
torch.cuda.synchronize()
print(f'H2D of {nbytes / 1e6:.1f} MB from pinned memory: {e0.elapsed_time(e1) / 5:.3f} ms = {nbytes * 5 / e0.elapsed_time(e1) / 1e6:.1f} GB/s')
del hp, dp

run(8)
print('per-call ms', [round(x, 2) for x in run(6, trace=True)])
ts = run(20)
print(f'   20 calls: median {np.median(ts):6.2f} ms  min {min(ts):6.2f}')
if os.environ.get('VPB_TIMELINE_SWEEP', '1') == '0':
    sys.exit(0)
for rows, sl, thr, mb in [(128, 8, 8, 256), (64, 8, 8, 256), (64, 16, 8, 256), (32, 8, 8, 256), (128, 8, 4, 256), (128, 4, 8, 256), (128, 16, 8, 256)]:
    MVectorPredictor.STAGE_ROWS, MVectorPredictor.COPY_SLICE, MVectorPredictor.MAX_BATCH = rows, sl, mb
    os.environ['VPB_GATHER_THREADS'] = str(thr)
    run(3)
    ts = run(8)
    print(f'STAGE_ROWS={rows:3d} COPY_SLICE={sl:2d} threads={thr:2d} MAX_BATCH={mb:3d}: median {np.median(ts):6.2f} ms  min {min(ts):6.2f}')
