"""FLAC decoding on the device (csrc/flac.cu): kernel time of vp_flac_decode on 256 x 3 s 16 kHz mono and 256 x 3 s
44.1 kHz stereo (CUDA events over many launches; one 3 s stream written by the test encoder, FIXED order 2 with Rice
partitions, repeated 256 times), with the compressed bytes in and samples out; beside it the front-end of the same
256 x 3 s 16 kHz batch (Fbank), and predict_batch end to end from the FLAC bytes against the same audio as float32
arrays, outputs compared; one hour at 16 kHz in one stream (a 10 s encoded chunk's frames repeated under new frame
numbers); evaluate over 64 synthetic 3 s files as FLAC and as 16-bit WAV, results compared.

Card name and power limit are read in the same run.  Usage: python tools/flac_times.py [--reps 50] [--out file.json]"""
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


def stream(rate, ch, seconds, seed):
    import flac_writer as fw
    rng = np.random.default_rng(seed)
    n = int(rate * seconds)
    t = np.arange(n)[:, None]
    x = 6000 * np.sin(2 * np.pi * t * rng.uniform(0.001, 0.05, size=(1, ch))) + rng.normal(0, 800, size=(n, ch))
    pcm = np.clip(np.round(x), -32768, 32767).astype(np.int64)
    return fw.encode(pcm, rate, 16, blocksize=4096, assign=(lambda fi: 10) if ch == 2 else None,
                     sub=lambda fi, c, x: dict(kind='fixed', order=2, part_order=4 if len(x) % 16 == 0 else 0))


def hour_stream():
    import flac_writer as fw
    from test_gpu_flac import _crc16_many
    rng = np.random.default_rng(7)
    bs, chunk = 4000, 160000
    t = np.arange(chunk)[:, None]
    x = 6000 * np.sin(2 * np.pi * t * 0.01) + rng.normal(0, 800, size=(chunk, 1))
    pcm = np.clip(np.round(x), -32768, 32767).astype(np.int64)
    tails = []
    fw.encode(pcm, 16000, 16, blocksize=bs, sub=lambda fi, c, x: dict(kind='fixed', order=2, part_order=4),
              frames_out=tails)
    n = 3600 * 16000
    si = dict(rate=16000, bps=16)
    bodies = []
    for f in range(n // bs):
        body = fw.frame_header(bs, f * bs, f, 0, 0, si) + tails[f % len(tails)][:-2]
        bodies.append(np.frombuffer(body, dtype=np.uint8))
    crcs = _crc16_many(bodies)
    frames = b''.join(b.tobytes() + int(c).to_bytes(2, 'big') for b, c in zip(bodies, crcs))
    return b'fLaC' + bytes([0x80, 0, 0, 34]) + fw._streaminfo(bs, bs, 0, 0, 16000, 1, 16, n) + frames


def evaluate_times(tmp):
    """evaluate over 64 synthetic 3 s files (16 distinct, 44.1 / 16 kHz) as FLAC and as 16-bit WAV: wall time of
    each and whether (eer, min_dcf, threshold) are equal."""
    import wave
    from mvector.trainer import MVectorTrainer
    from oracle import models as om
    margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
    out = {}
    pcms = []
    rng = np.random.default_rng(9)
    for i in range(16):
        rate = (16000, 44100)[i % 2]
        pcms.append((np.clip(np.round(6000 * np.sin(2 * np.pi * np.arange(3 * rate) * rng.uniform(0.001, 0.05))
                                      + rng.normal(0, 800, 3 * rate)), -32768, 32767).astype(np.int64), rate))
    import flac_writer as fw
    encoded = [fw.encode(p, r, 16, blocksize=4096, sub=lambda fi, c, x: dict(kind='fixed', order=2)) for p, r in pcms]
    for fmt in ('flac', 'wav'):
        os.makedirs(os.path.join(tmp, fmt))
        lines = []
        for i in range(64):
            p = os.path.join(tmp, fmt, f'{i}.{fmt}')
            pcm, rate = pcms[i % 16]
            if fmt == 'flac':
                open(p, 'wb').write(encoded[i % 16])
            else:
                with wave.open(p, 'wb') as w:
                    w.setnchannels(1); w.setsampwidth(2); w.setframerate(rate); w.writeframes(pcm.astype('<i2').tobytes())
            lines.append(f'{p}\t{i % 8}\n')
        lst = os.path.join(tmp, fmt, 'list.txt')
        open(lst, 'w').write(''.join(lines))
        cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                            'use_dB_normalization': True, 'target_dB': -20},
                                'eval_conf': {'batch_size': 32, 'max_duration': 20}, 'train_list': lst,
                                'enroll_list': lst, 'trials_list': lst},
               'preprocess_conf': {'feature_method': 'Fbank', 'method_args': dict(sample_frequency=16000, num_mel_bins=80)},
               'model_conf': {'model': 'EcapaTdnn', 'model_args': margs}}
        tr = MVectorTrainer(cfg, use_gpu=True)
        tr._setup_eval()
        tr.model.load_state_dict(om.random_state_dict('EcapaTdnn', 80, seed=0, **margs))
        tr.evaluate()
        s = time.perf_counter()
        r = tr.evaluate()
        out[fmt] = dict(seconds=round(time.perf_counter() - s, 3), result=[float(v) for v in r])
    out['equal'] = out['flac']['result'] == out['wav']['result']
    return out


def main():
    import __graft_entry__ as ge
    ge.build()
    from mvector.engine import Engine
    from mvector.flac import FlacBatch, parse_streaminfo
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    eng = Engine(0)
    res = {'card': card(), 'decode': []}
    for rate, ch in ((16000, 1), (44100, 2)):
        data = stream(rate, ch, 3.0, seed=rate + ch)
        si = parse_streaminfo(data)
        batch = FlacBatch([data] * 256, [si] * 256, eng.device)
        out = torch.empty(256, si.total_samples, dtype=torch.float32, device=eng.device)
        status = torch.empty(256, dtype=torch.int32, device=eng.device)
        ms = event_ms(lambda: eng.decode_flac_into(batch, out, si.total_samples, status), a.reps)
        assert not status.cpu().numpy().any()
        res['decode'].append(dict(rate=rate, channels=ch, items=256, seconds=3.0, bytes_in=batch.nbytes,
                                  samples_out=256 * si.total_samples * ch, pcm_float32_bytes=256 * si.total_samples * 4,
                                  kernel_ms=round(ms, 4)))
        print(res['decode'][-1], flush=True)

    # one hour at 16 kHz: a 10 s encoded chunk's frames repeated with new frame numbers
    data = hour_stream()
    si = parse_streaminfo(data)
    batch = FlacBatch([data], [si], eng.device)
    out = torch.empty(1, si.total_samples, dtype=torch.float32, device=eng.device)
    status = torch.empty(1, dtype=torch.int32, device=eng.device)
    ms = event_ms(lambda: eng.decode_flac_into(batch, out, si.total_samples, status), 3)
    assert not status.cpu().numpy().any()
    res['decode'].append(dict(rate=16000, channels=1, items=1, seconds=3600.0, bytes_in=batch.nbytes,
                              samples_out=si.total_samples, pcm_float32_bytes=si.total_samples * 4,
                              kernel_ms=round(ms, 4)))
    print(res['decode'][-1], flush=True)

    # the front-end of the same 16 kHz batch, and predict_batch end to end
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
    distinct = [stream(16000, 1, 3.0, seed=100 + i) for i in range(16)]      # the Python encoder is slow
    datas = [distinct[i % 16] for i in range(256)]
    rows, _ = pred._engine.decode_flac(datas)
    arrays = [r.copy() for r in rows.cpu().numpy()]
    from mvector.data_utils.featurizer import AudioFeaturizer
    fz = AudioFeaturizer('Fbank', method_args=dict(sample_frequency=16000, num_mel_bins=80), engine=pred._engine)
    wave = rows.contiguous()
    res['fbank_ms_256x3s_16k'] = round(event_ms(lambda: fz(wave), a.reps), 4)

    def wall(fn, reps=5):
        fn()
        t = []
        for _ in range(reps):
            s = time.perf_counter()
            fn()
            t.append((time.perf_counter() - s) * 1e3)
        return round(float(np.median(t)), 3)
    e_flac, e_arr = pred.predict_batch(datas), pred.predict_batch(arrays)
    res['predict_batch'] = dict(items=256, flac_ms=wall(lambda: pred.predict_batch(datas)),
                                float32_ms=wall(lambda: pred.predict_batch(arrays)),
                                equal=bool(np.array_equal(e_flac, e_arr)))
    with tempfile.TemporaryDirectory() as td:
        res['evaluate_64_files'] = evaluate_times(td)
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
