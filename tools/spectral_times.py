"""Time the diarization clustering's spectral stage on the device against the host path, in one run.

For every n (chunks of a recording; 0.75 s apart, so n = 3200 is 40 minutes) on seeded 6-speaker synthetic 192-d
embeddings:
  * each device stage with CUDA events around it and a synchronise: Laplacian (vp_spectral_laplacian), Householder
    reduction (vp_sym_tridiag), back-transformation (vp_sym_tridiag_apply_q, with the [n, k] upload and download);
  * the host tridiagonal solve (LAPACK stebz / stein through scipy) with the d, e download;
  * SpectralCluster.__call__ with the device hook and without it (the host path: float32 cosine, argsort pruning,
    dense scipy.linalg.eigh, k-means), wall clock;
  * the pass's achieved HBM rate from the bytes it moves by shape (read + write of the m x m trailing block per step,
    read only at the first step): over the whole reduction's event time (a lower bound), and over the pass kernels'
    own summed time from torch.profiler in a subprocess with VPB_PDL=0 -- with programmatic dependent launch a kernel
    starts early and waits, so profiled kernel durations overlap and only the serialised run splits the time
    between pass and reflector kernels.
Prints one line per n and the card (name, power limit, max SM clock from a read-only nvidia-smi query) and host core
count; --out writes the same as JSON.

    python tools/spectral_times.py [--sizes 500,1000,2000,3200,4800,8000] [--host-max-n N] [--out times.json]
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


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown (nvidia-smi failed)'


def embeddings(n, spk=6, dim=192, seed=0):
    rng = np.random.RandomState(seed)
    cen = rng.randn(spk, dim)
    turn = np.repeat(rng.randint(0, spk, n // 8 + 1), 8)[:n]
    x = cen[turn] + 0.5 * rng.randn(n, dim)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def pass_bytes(n):
    m = np.arange(n - 1, 1, -1, dtype=np.float64)          # trailing block of steps k = 0 .. n-3
    return float(8 * (m ** 2).sum() * 2 - 8 * (n - 1) ** 2)  # read + write, the first step only reads


def profile_serialised(n):
    """(summed pass kernel ms, summed reflector kernel ms, event ms) of one vp_sym_tridiag at size n; run with
    VPB_PDL=0 so that kernels do not overlap."""
    import torch
    from mvector.engine import Engine
    from mvector.infer_utils.speaker_diarization import SpectralCluster
    eng = Engine()
    X = embeddings(n)
    nd = SpectralCluster().n_drop(n)
    scratch = eng.spectral_scratch(n)
    eng.sym_tridiag(eng.spectral_laplacian(X, nd, scratch), scratch)                # warm-up
    A = eng.spectral_laplacian(X, nd, scratch)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ev[0].record()
        eng.sym_tridiag(A, scratch)
        ev[1].record()
        torch.cuda.synchronize()
    k_pass = k_refl = 0.0
    for evt in prof.events():
        if evt.device_type == torch.autograd.DeviceType.CUDA:
            if 'tridiag_pass_kernel' in evt.name:
                k_pass += evt.device_time_total / 1e3
            elif 'reflect_kernel' in evt.name:
                k_refl += evt.device_time_total / 1e3
    eng.close()
    return k_pass, k_refl, ev[0].elapsed_time(ev[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='500,1000,2000,3200,4800,8000')
    ap.add_argument('--out', default=None)
    ap.add_argument('--host-max-n', type=int, default=0,
                    help='skip the host path above this n (0: never); its dense eigh takes minutes at n = 8000')
    ap.add_argument('--profile-serialised', type=int, default=0, help=argparse.SUPPRESS)
    args = ap.parse_args()
    import __graft_entry__
    __graft_entry__.build()
    import scipy.linalg
    import torch
    from mvector import _lib as L
    from mvector.engine import Engine
    from mvector.infer_utils.speaker_diarization import SpectralCluster
    assert torch.cuda.is_available(), 'spectral_times.py measures the device: it needs a GPU'
    if args.profile_serialised:
        print(json.dumps(profile_serialised(args.profile_serialised)))
        return
    eng = Engine()
    info = dict(card=card(), host_cores=os.cpu_count(), torch=torch.__version__)
    print(f"card: {info['card']}  host cores: {info['host_cores']}")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def timed(fn):
        torch.cuda.synchronize()
        ev[0].record()
        out = fn()
        ev[1].record()
        torch.cuda.synchronize()
        return out, ev[0].elapsed_time(ev[1])

    sc = SpectralCluster()
    rows = []
    # warm-up: module load, allocator, every kernel once, k-means and LAPACK on both paths
    X = embeddings(300)
    warm = SpectralCluster()
    warm.spectral_fn = eng.spectral_embedding
    warm(X)
    SpectralCluster()(X)
    for n in [int(s) for s in args.sizes.split(',')]:
        X = embeddings(n)
        nd, n_eig = sc.n_drop(n), min(n, sc.max_num_spks + 1)
        scratch = eng.spectral_scratch(n)
        A, t_lap = timed(lambda: eng.spectral_laplacian(X, nd, scratch))
        (d, e, tau), t_tri = timed(lambda: eng.sym_tridiag(A, scratch))
        t0 = time.perf_counter()
        dh, eh = d.cpu().numpy(), e.cpu().numpy()
        lam = scipy.linalg.eigh_tridiagonal(dh, eh, eigvals_only=True, select='i', select_range=(0, n_eig - 1))
        k = sc.num_speakers(lam)
        _, Zt = scipy.linalg.eigh_tridiagonal(dh, eh, select='i', select_range=(0, k - 1))
        t_host_tri = (time.perf_counter() - t0) * 1e3
        Z, t_q = timed(lambda: eng.sym_tridiag_apply_q(A, tau, Zt).cpu())
        # SpectralCluster end to end, device hook vs host path, same seed
        dev = SpectralCluster()
        dev.spectral_fn = eng.spectral_embedding
        np.random.seed(0)
        t0 = time.perf_counter()
        lab_dev = dev(X.copy())
        t_dev_call = (time.perf_counter() - t0) * 1e3
        lab_host, t_host_call = None, float('nan')
        if not args.host_max_n or n <= args.host_max_n:
            np.random.seed(0)
            t0 = time.perf_counter()
            lab_host = SpectralCluster()(X.copy())
            t_host_call = (time.perf_counter() - t0) * 1e3
        r = subprocess.run([sys.executable, os.path.abspath(__file__), '--profile-serialised', str(n)],
                           env=dict(os.environ, VPB_PDL='0'), capture_output=True, text=True, cwd=ROOT)
        assert r.returncode == 0, r.stderr[-2000:]
        k_pass, k_refl, t_tri_serial = json.loads(r.stdout.strip().splitlines()[-1])
        pb = pass_bytes(n)
        row = dict(n=n, launches=int(L.lib().vp_spectral_launches(n)), k=int(k),
                   laplacian_ms=t_lap, tridiag_ms=t_tri, host_tridiag_solve_ms=t_host_tri, apply_q_ms=t_q,
                   device_stage_ms=t_lap + t_tri + t_host_tri + t_q,
                   cluster_call_device_ms=t_dev_call, cluster_call_host_ms=t_host_call,
                   speedup_call=t_host_call / t_dev_call,
                   pass_bytes=pb, pass_TBps_over_tridiag=pb / (t_tri * 1e-3) / 1e12,
                   serialised_tridiag_ms=t_tri_serial, pass_kernels_ms=k_pass, reflect_kernels_ms=k_refl,
                   pass_TBps=pb / (k_pass * 1e-3) / 1e12 if k_pass > 0 else None,
                   labels_equal=None if lab_host is None else bool(np.array_equal(lab_dev, lab_host)))
        rows.append(row)
        print(f"n={n:5d} launches={row['launches']:6d} k={k:2d} | laplacian {t_lap:8.2f} ms  tridiag {t_tri:9.2f} ms  "
              f"host tridiag solve+copy {t_host_tri:7.2f} ms  apply_q {t_q:7.2f} ms | SpectralCluster device "
              f"{t_dev_call:9.1f} ms  host {t_host_call:9.1f} ms  ({row['speedup_call']:.1f}x, labels equal "
              f"{row['labels_equal']}) | pass {pb / 1e9:7.1f} GB: {row['pass_TBps_over_tridiag']:.2f} TB/s over the "
              f"reduction; serialised (VPB_PDL=0) reduction {t_tri_serial:8.2f} ms = pass kernels {k_pass:8.2f} ms "
              f"({row['pass_TBps'] or 0:.2f} TB/s) + reflect kernels {k_refl:7.2f} ms + gaps", flush=True)
        del A, Z, scratch
        torch.cuda.empty_cache()
    eng.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(dict(info=info, rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
