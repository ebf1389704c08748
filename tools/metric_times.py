"""Time evaluate's verification metrics on the device (csrc/verify.cu) against the host path, in one run.

For every N = n_trials * n_enroll (trial-major matrix form, seeded normal scores, 400 speakers):
  * Engine.verification_metrics end to end (scores already on the device; includes the result copy and its
    synchronise), CUDA events, median of --reps calls after a warm-up;
  * each of the four radix-sort passes (histogram + 3-launch scan + scatter) and the curve pass (counts + scan +
    evaluation + final reduction), summed kernel durations from torch.profiler in a subprocess with VPB_PDL=0 -- with
    programmatic dependent launch a kernel starts early and waits, so only a serialised run splits the time;
  * the bytes each pass moves by shape and the achieved TB/s;
  * the host path (np.argsort + compute_fnr_fpr / compute_eer / compute_dcf on the same scores and the int32 label
    matrix), wall clock, up to 2^--host-max-log2.
Prints the card (name, power limit, max SM clock from a read-only nvidia-smi query) and one line per N; --out writes
JSON.

    python tools/metric_times.py [--log2 20,22,24,26,28] [--host-max-log2 24] [--reps 5] [--out times.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TILE = 4096


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown (nvidia-smi failed)'


def problem(k, seed=0):
    nt, ne = 1 << ((k + 1) // 2), 1 << (k // 2)
    rng = np.random.RandomState(seed)
    return nt, ne, rng.randint(0, 400, nt).astype(np.int32), rng.randint(0, 400, ne).astype(np.int32)


def device_scores(nt, ne, seed=0):
    import torch
    g = torch.Generator(device='cuda').manual_seed(seed)
    return torch.randn(nt * ne, generator=g, device='cuda', dtype=torch.float32) * 0.3


def pass_bytes(n):
    """Bytes each stage moves by shape: sort pass p (p = 0 reads the fp32 scores and forms keys and labels from the
    small label vectors), and the curve pass."""
    nt = -(-n // TILE)
    scan = 4 * 256 * nt * 4                                  # histogram write, chunk-sum read, down-sweep read + write
    sort = [4 * n + (4 * n + 4 * n + n) + scan]              # hist read | scatter: read keys, write keys + labels
    sort += [4 * n + (5 * n + 5 * n) + scan] * 3
    curve = n + n                                            # counts read, evaluation read
    return sort, curve


def profile(k):
    """Summed kernel ms of [sort pass 0..3, curve pass] for one call at N = 2^k (run with VPB_PDL=0)."""
    import torch
    from mvector.engine import Engine
    eng = Engine()
    nt, ne, tl, el = problem(k)
    s = device_scores(nt, ne)
    eng.verify(s, trial_labels=tl, enroll_labels=el)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.verify(s, trial_labels=tl, enroll_labels=el)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
                 and any(t in e.name for t in ('radix_', 'scan_', 'curve_'))), key=lambda e: e.time_range.start)
    names = [e.name for e in ev]
    assert len(ev) == 26, names                              # 4 x (hist + 3 scan + scatter) + count + 3 scan + eval + final
    dur = [e.time_range.elapsed_us() / 1e3 for e in ev]
    return [sum(dur[5 * p:5 * p + 5]) for p in range(4)] + [sum(dur[20:])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--log2', default='20,22,24,26,28')
    ap.add_argument('--host-max-log2', type=int, default=24)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out')
    ap.add_argument('--profile-one', type=int, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.profile_one is not None:
        print(json.dumps(profile(a.profile_one)))
        return
    import torch
    from mvector.engine import Engine
    from mvector.metric.metrics import compute_dcf, compute_eer, compute_fnr_fpr
    assert torch.cuda.is_available(), 'metric_times.py measures on the GPU'
    eng = Engine()
    print(f'card: {card()}; host cores: {os.cpu_count()}')
    rows = []
    for k in [int(x) for x in a.log2.split(',')]:
        nt, ne, tl, el = problem(k)
        n = nt * ne
        s = device_scores(nt, ne)
        out = eng.verification_metrics(s, trial_labels=tl, enroll_labels=el)           # warm-up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            e0.record()
            eng.verification_metrics(s, trial_labels=tl, enroll_labels=el)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        env = dict(os.environ, VPB_PDL='0')
        r = subprocess.run([sys.executable, os.path.abspath(__file__), '--profile-one', str(k)], env=env,
                           capture_output=True, text=True)
        passes = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else None
        if passes is None:
            sys.stderr.write(r.stderr[-2000:])
        sb, cb = pass_bytes(n)
        row = dict(log2=k, n=n, n_trials=nt, n_enroll=ne, device_ms=float(np.median(ms)), eer=out[0], min_dcf=out[1],
                   pass_ms=passes, pass_gb=[b / 1e9 for b in sb + [cb]])
        if passes:
            row['pass_tbs'] = [b / (t * 1e-3) / 1e12 for b, t in zip(sb + [cb], passes)]
        if k <= a.host_max_log2:
            host = s.cpu().numpy()
            t0 = time.perf_counter()
            lab = (tl[:, None] == el[None, :]).astype(np.int32).reshape(-1)
            fnr, fpr, _ = compute_fnr_fpr(host, lab)
            compute_eer(fnr, fpr, host)
            compute_dcf(fnr, fpr)
            row['host_s'] = time.perf_counter() - t0
        rows.append(row)
        ps = ' '.join(f'{t:.3f}ms/{r_:.2f}TB/s' for t, r_ in zip(passes, row['pass_tbs'])) if passes else 'not measured'
        hs = f"{row['host_s']:.3f} s" if 'host_s' in row else 'not measured'
        print(f"N=2^{k} ({nt}x{ne}): device {row['device_ms']:.3f} ms end to end; passes (sort 0-3, curve): {ps}; "
              f"GB by shape {sum(row['pass_gb']):.2f}; host path {hs}", flush=True)
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
