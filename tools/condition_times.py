"""Input conditioning (resample + dB normalisation, csrc/condition.cu) inside predict_batch: EcapaTdnn + Fbank, 256 x 3 s
per call, use_dB_normalization on, inputs at 16 / 8 / 44.1 / 48 kHz.  Per rate:

  * e2e: predict_batch on the native-rate arrays (device conditioning), median ms after warm-up, ending in the host result;
  * host: the same list conditioned on the host (AudioSegment.resample + normalize, the former per-item path), median ms,
    and a normalisation-off predictor on those inputs (what the device path must equal);
  * kernels: vp_resample and vp_gain_normalize alone on the [256, native] device batch, CUDA events over many launches;
  * bytes and fp64 FLOPs of the two kernels by shape.

Card name and power limit are read in the same run.  Usage: python tools/condition_times.py [--reps 20] [--out file.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001
        return f'unknown ({e})'


def median_ms(fn, reps, sync=True):
    out = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        if sync:
            torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1e3)
    return float(np.median(out))


def event_ms(fn, reps):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    assert torch.cuda.is_available(), 'condition_times measures on the GPU'
    from mvector.audio import AudioSegment, polyphase_taps, resample_ratio
    from mvector.predict import MVectorPredictor
    from oracle import models as om
    margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
    sd = om.random_state_dict('EcapaTdnn', 80, seed=0, **margs)

    def predictor(db):
        cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                            'use_dB_normalization': db, 'target_dB': -20},
                                'eval_conf': {'batch_size': 16, 'max_duration': 20}},
               'preprocess_conf': {'use_hf_model': False, 'feature_method': 'Fbank',
                                   'method_args': dict(sample_frequency=16000, num_mel_bins=80)},
               'model_conf': {'model': 'EcapaTdnn', 'model_args': dict(margs)}}
        with tempfile.TemporaryDirectory() as td:
            torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
            return MVectorPredictor(configs=cfg, model_path=td, use_gpu=True)

    pn, pp = predictor(True), predictor(False)
    eng = pn._engine
    B = args.batch
    rows = []
    for sr in (16000, 8000, 44100, 48000):
        g = torch.Generator().manual_seed(sr)
        waves = [(torch.randn(3 * sr, generator=g) * 0.1).numpy() for _ in range(B)]

        def host_condition():
            out = []
            for w in waves:
                seg = AudioSegment(w, sr)
                seg.resample(16000)
                seg.normalize(target_db=-20)
                out.append(seg.samples)
            return out
        for _ in range(2):
            dev = pn.predict_batch(waves, sample_rate=sr)
        e2e = median_ms(lambda: pn.predict_batch(waves, sample_rate=sr), args.reps)
        t = time.perf_counter()
        hosted = host_condition()
        host_ms = (time.perf_counter() - t) * 1e3
        for _ in range(2):
            ref = pp.predict_batch(hosted)
        off = median_ms(lambda: pp.predict_batch(hosted), args.reps)
        # kernels alone on the device batch
        up, down = resample_ratio(sr, 16000)
        x = torch.from_numpy(np.stack(waves)).cuda()
        n_in = [3 * sr] * B
        rs = eng.condition_plan(n_in, sr, 16000)                         # resample only
        lout = int(rs.n_out.max())
        y = torch.zeros(B, lout, dtype=torch.float32, device='cuda')
        rs_ms = event_ms(lambda: rs.run(x, x.shape[1], y, lout, 0, B, None, None), 50) if rs.resample else None
        if not rs.resample:
            y.copy_(x)
        gn = eng.condition_plan([lout] * B, 16000, 16000, -20.0)           # gain only, on the 16 kHz rows
        flags = torch.empty(B, dtype=torch.int32, device='cuda')
        scratch = gn.scratch(B, lout)
        gain_ms = event_ms(lambda: gn.run(y, lout, y, lout, 0, B, flags, scratch), 50)
        nt = polyphase_taps(up, down)[1] if up != down else 0             # taps per output (one phase row)
        rows.append(dict(
            rate=sr, up=up, down=down, taps_per_output=nt, n_in=3 * sr, n_out=lout,
            e2e_device_conditioned_ms=e2e, host_conditioning_ms=host_ms, e2e_host_conditioned_inputs_norm_off_ms=off,
            equal_to_host_conditioned=bool(np.array_equal(dev, ref)),
            resample_kernel_ms=rs_ms, gain_kernels_ms=gain_ms,
            resample_bytes=(B * 3 * sr + B * lout) * 4 if up != down else 0, resample_fp64_flop=2.0 * B * lout * nt,
            gain_bytes=B * lout * 4 * 3, gain_fp64_flop=B * lout * 4.0))
        print(json.dumps(rows[-1]), flush=True)
    res = dict(card=card(), batch=B, seconds=3, model='EcapaTdnn+Fbank80', rows=rows)
    print(json.dumps(dict(card=res['card'])))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
