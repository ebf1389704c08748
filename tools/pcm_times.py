"""PCM container conversion on the device (csrc/pcm.cu): CUDA-event time of vp_pcm_decode, with the bytes it reads and
writes, on 256 x 3 s 16 kHz mono 16-bit WAV, 256 x 3 s 44.1 kHz stereo 24-bit WAV and one hour of 16 kHz mono 16-bit
WAV; then predict_batch end to end on 256 16-bit WAV files three ways: the standard-library ``wave`` reader with a numpy
conversion and host staging (the path these files took before PcmSegment; AudioSegment._from_wave is still that
reader), the new path (the files' bytes go up in one pinned copy and each stage converts on the device), and the same
audio as float32 arrays; outputs compared.  Wall-clock medians after a warm-up call.

Card name and power limit are read in the same run.  Usage: python tools/pcm_times.py [--reps 50] [--out file.json]"""
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
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001
        return f'unknown ({e})'


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def wall(fn, reps=5):
    fn()
    t = []
    for _ in range(reps):
        s = time.perf_counter()
        fn()
        t.append((time.perf_counter() - s) * 1e3)
    return round(float(np.median(t)), 3)


def speech(rate, ch, seconds, seed):
    rng = np.random.default_rng(seed)
    n = int(rate * seconds)
    t = np.arange(n)[:, None]
    x = 6000 * np.sin(2 * np.pi * t * rng.uniform(0.001, 0.05, size=(1, ch))) + rng.normal(0, 800, size=(n, ch))
    return np.clip(np.round(x), -32768, 32767).astype(np.int64)


def wav_file(ints, rate, fmt):
    import pcm_writer as pw
    vals = ints.reshape(-1) << (8 if fmt == 's24le' else 0)
    return pw.wav(pw.encode(vals, fmt), rate, ints.shape[1], fmt)


def kernel(eng, files, reps, label):
    from mvector.pcm import PcmBatch, parse_header
    infos = [parse_header(f) for f in files]
    batch = PcmBatch(files, infos, eng.device)
    ld = max(i.frames for i in infos)
    out = torch.empty(len(files), ld, dtype=torch.float32, device=eng.device)
    status = torch.empty(len(files), dtype=torch.int32, device=eng.device)
    ms = event_ms(lambda: eng.decode_pcm_into(batch, out, ld, status), reps)
    assert not status.cpu().numpy().any()
    read = sum(i.frames * i.channels * i.width for i in infos)
    written = len(files) * ld * 4
    r = dict(input=label, rows=len(files), bytes_read=read, bytes_written=written, kernel_us=round(ms * 1e3, 2),
             tb_per_s=round((read + written) / (ms * 1e-3) / 1e12, 3))
    print(r, flush=True)
    return r


def main():
    import __graft_entry__ as ge
    ge.build()
    from mvector.audio import AudioSegment
    from mvector.engine import Engine
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    eng = Engine(0)
    res = {'card': card(), 'decode': []}
    mono16 = [wav_file(speech(16000, 1, 3.0, seed=i), 16000, 's16le') for i in range(256)]
    res['decode'].append(kernel(eng, mono16, a.reps, '256 x 3 s 16 kHz mono 16-bit'))
    stereo24 = [wav_file(speech(44100, 2, 3.0, seed=i), 44100, 's24le') for i in range(256)]
    res['decode'].append(kernel(eng, stereo24, a.reps, '256 x 3 s 44.1 kHz stereo 24-bit'))
    hour = wav_file(np.tile(speech(16000, 1, 10.0, seed=7), (360, 1)), 16000, 's16le')
    res['decode'].append(kernel(eng, [hour], 10, '1 h 16 kHz mono 16-bit'))

    from mvector.predict import MVectorPredictor
    from oracle import models as om
    margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
    sd = om.random_state_dict('EcapaTdnn', 80, seed=0, **margs)
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                            'use_dB_normalization': True, 'target_dB': -20},
                                'eval_conf': {'batch_size': 16, 'max_duration': 20}},
               'preprocess_conf': {'use_hf_model': False, 'feature_method': 'Fbank',
                                   'method_args': dict(sample_frequency=16000, num_mel_bins=80)},
               'model_conf': {'model': 'EcapaTdnn', 'model_args': margs}}
        pred = MVectorPredictor(configs=cfg, model_path=td, use_gpu=True)
    with tempfile.TemporaryDirectory() as td:
        paths = []
        for i, d in enumerate(mono16):
            paths.append(os.path.join(td, f'{i}.wav'))
            with open(paths[-1], 'wb') as f:
                f.write(d)
        arrays = [AudioSegment.from_file(p).samples for p in paths]

        def before():           # the wave reader, numpy conversion and host staging
            return pred.predict_batch([AudioSegment._from_wave(p) for p in paths])
        e_new, e_old, e_arr = pred.predict_batch(paths), before(), pred.predict_batch(arrays)
        res['predict_batch'] = dict(items=256, wav_files='3 s 16 kHz mono 16-bit',
                                    before_wave_host_ms=wall(before), after_device_ms=wall(lambda: pred.predict_batch(paths)),
                                    float32_arrays_ms=wall(lambda: pred.predict_batch(arrays)),
                                    equal=bool(np.array_equal(e_new, e_old) and np.array_equal(e_new, e_arr)))
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
