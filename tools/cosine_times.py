"""Time the cosine score kernel (csrc/pool.cu cosine_scores_kernel through vp_cosine_scores) at the sizes its callers
run: an evaluate trial x enrol matrix (4708 x 4708 x 192), a diarization affinity (2500 x 2500 x 192), retrieval of a
batch of 256 queries against 1000 enrolled speakers, and 2,097,121 x 3 x 4 (more tile rows than one grid column holds).

Inputs and output are preallocated on the device, so each timed call is one kernel launch.  Per shape: the median of
--reps CUDA-event timings of --inner back-to-back calls, after a warm-up; the dot-product FLOPs (2 n m D) and the
compulsory bytes (4 (n D + m D + n m)) by shape, and the rates they give.  Prints the card (name, power limit, max SM
clock) and one line per shape, or the error of a build that refuses the shape; --out writes JSON.  VPB_LIB selects
another build of the library, so two builds can be compared by running this script once with each.

    python tools/cosine_times.py [--reps 7] [--inner 20] [--out times.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [('evaluate', 4708, 4708, 192), ('diarization', 2500, 2500, 192), ('retrieval', 256, 1000, 192),
          ('tall', 65535 * 32 + 1, 3, 4)]


def card():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'unknown (nvidia-smi failed)'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=7)
    ap.add_argument('--inner', type=int, default=20)
    ap.add_argument('--out')
    args = ap.parse_args()
    import torch
    from mvector import _lib as L
    from mvector.engine import Engine
    eng = Engine()
    lib, stream = L.lib(), eng.stream_ptr()
    g = torch.Generator(device='cuda').manual_seed(0)
    rows = []
    print(f'card: {card()}  library: {L.LIB_PATH}')
    for name, n, m, D in SHAPES:
        a = torch.randn(n, D, generator=g, device='cuda')
        b = torch.randn(m, D, generator=g, device='cuda')
        out = torch.empty(n, m, device='cuda')

        def call():
            rc = lib.vp_cosine_scores(eng.handle, C.c_void_p(a.data_ptr()), n, C.c_void_p(b.data_ptr()), m, D,
                                      C.c_void_p(out.data_ptr()), stream)
            if rc != L.VP_OK:
                raise L.VpError(rc, lib.vp_last_error(eng.handle).decode())

        try:
            for _ in range(3):
                call()
            torch.cuda.synchronize()
        except L.VpError as e:                       # a build that cannot launch this shape
            print(f'{name:12s} {n:8d} x {m:5d} x {D:4d}: refused: {e}')
            rows.append(dict(name=name, n=n, m=m, D=D, error=str(e)))
            continue
        times = []
        for _ in range(args.reps):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.inner):
                call()
            t1.record()
            t1.synchronize()
            times.append(t0.elapsed_time(t1) / args.inner)
        times.sort()
        ms = times[len(times) // 2]
        flop, nbytes = 2.0 * n * m * D, 4.0 * (n * D + m * D + n * m)
        row = dict(name=name, n=n, m=m, D=D, ms=ms, ms_min=times[0], ms_max=times[-1],
                   tflops=flop / ms * 1e-9, tb_s=nbytes / ms * 1e-9)
        rows.append(row)
        print(f'{name:12s} {n:8d} x {m:5d} x {D:4d}: {ms:8.4f} ms (min {times[0]:.4f}, max {times[-1]:.4f})  '
              f'{row["tflops"]:6.2f} TFLOP/s dot  {row["tb_s"]:5.3f} TB/s compulsory')
        del a, b, out
    eng.close()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=card(), library=L.LIB_PATH, rows=rows), f, indent=1)


if __name__ == '__main__':
    main()
