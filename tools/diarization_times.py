"""speaker_diarization on one long recording: the device front (one upload at the native rate, device conditioning, frame
energies and chunk windows) against the host flow it replaced, reconstructed from the public pieces
(_condition_host -> segments_audio -> predict_batch -> clustering -> postprocess).

Seeded synthetic recordings of four speakers taking turns (harmonic voices in noise, with pauses), 10 and 60 minutes at
16 and 44.1 kHz; CAM++ (CAMPPlus, embd_dim 192, 80-bin Fbank at 16 kHz, dB normalisation on: configs/cam++.yml) with
seeded random weights.  Per recording:

  * wall-clock median of whole calls after one warm-up, new path and host flow, and whether their outputs are equal;
  * CUDA-event times of the new path's stages, run one after another: upload, conditioning, frame energies, the gather
    of every chunk row (alone; inside the embedding it runs per stage on the copy stream), embedding of the chunks
    (staging + front-end + backbone) and the spectral stage of the clustering.

Card name and power limit are read in the same run.  Usage:
  python tools/diarization_times.py [--minutes 10 60] [--rates 16000 44100] [--reps 2] [--out file.json]"""
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


def recording(minutes, sr, seed=0):
    """Four speakers (f0 105 / 160 / 220 / 300 Hz, eight harmonics each, in noise) taking turns of 1-6 s with 0.2-1.5 s
    pauses, float32 at ``sr`` Hz."""
    rng = np.random.RandomState(seed)
    n = int(minutes * 60 * sr)
    x = (0.002 * rng.randn(n)).astype(np.float32)
    pos = int(0.5 * sr)
    while pos < n:
        d = min(int(rng.uniform(1.0, 6.0) * sr), n - pos)
        f0 = (105.0, 160.0, 220.0, 300.0)[rng.randint(4)] * rng.uniform(0.97, 1.03)
        t = np.arange(d) / float(sr)
        v = np.zeros(d)
        for h in range(1, 9):
            v += np.sin(2 * np.pi * f0 * h * t + rng.uniform(0, 2 * np.pi)) / h
        x[pos:pos + d] += (0.1 * v).astype(np.float32)
        pos += d + int(rng.uniform(0.2, 1.5) * sr)
    return x


def median_s(fn, reps):
    fn()
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t)
    return float(np.median(out)), out


def stage_ms(pred, x, sr):
    """CUDA-event times (ms) of the new path's stages, each synchronised before the next."""
    from mvector.audio import AudioSegment
    from mvector.predict import DeviceWindows
    eng = pred._engine
    ds = pred.configs.dataset_conf.dataset
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
    torch.cuda.synchronize()
    ev[0].record()
    xd = torch.from_numpy(x).to(pred.device)
    ev[1].record()
    y, n_out, _ = eng.condition(xd.view(1, -1), [x.size], [sr], ds.sample_rate, ds.target_dB)
    ev[2].record()
    n, msr = int(n_out[0]), int(ds.sample_rate)
    energy = eng.frame_energy(y.view(-1), n, AudioSegment.vad_hop(msr))
    ev[3].record()
    energy = energy.cpu().numpy()
    table = pred.speaker_diarize.chunk_table(AudioSegment.vad_from_energy(energy, n, msr, return_seconds=True), n, msr)
    wins = DeviceWindows(eng, y.view(-1), table)
    rows = torch.empty(len(wins), table.size, device=pred.device)
    torch.cuda.synchronize()
    ev[4].record()
    eng.gather_windows(wins.src, wins._offset, wins._valid, table.size, rows)
    ev[5].record()
    lmax = int(pred._output_lengths([table.size], [sr])[0])
    emb = pred._embed_waves(wins, lmax, masked=True, to_numpy=False, rates=[sr] * len(wins))
    ev[6].record()
    torch.cuda.synchronize()
    sc = pred.speaker_diarize.spectral_cluster
    B = emb.shape[0]
    feats = emb.cpu().numpy()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    eng.spectral_embedding(feats, sc.n_drop(B), min(B, sc.max_num_spks + 1), lambda lam: sc.num_speakers(lam, None))
    b.record()
    b.synchronize()
    out = dict(upload=ev[0].elapsed_time(ev[1]), condition=ev[1].elapsed_time(ev[2]), frame_energy=ev[2].elapsed_time(ev[3]),
               gather_all=ev[4].elapsed_time(ev[5]), embed=ev[5].elapsed_time(ev[6]), spectral=a.elapsed_time(b))
    out['chunks'] = B
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--minutes', type=float, nargs='+', default=[10, 60])
    ap.add_argument('--rates', type=int, nargs='+', default=[16000, 44100])
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    assert torch.cuda.is_available(), 'diarization_times measures on the GPU'
    from mvector.audio import AudioSegment
    from mvector.predict import MVectorPredictor
    from oracle import models as om
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': True, 'target_dB': -20},
                            'eval_conf': {'batch_size': 16, 'max_duration': 20}},
           'preprocess_conf': {'use_hf_model': False, 'feature_method': 'Fbank',
                               'method_args': dict(sample_frequency=16000, num_mel_bins=80)},
           'model_conf': {'model': 'CAMPPlus', 'model_args': dict(embd_dim=192)}}
    sd = om.random_state_dict('CAMPPlus', 80, seed=0, embd_dim=192)
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        pred = MVectorPredictor(configs=cfg, model_path=td, use_gpu=True)

    def host_flow(x, sr):
        seg = pred._condition_host(AudioSegment(x.copy(), sr))
        segments = pred.speaker_diarize.segments_audio(seg)
        feats = pred.predict_batch([s[2] for s in segments], sample_rate=sr)
        np.random.seed(0)
        labels, _ = pred.speaker_diarize.clustering(feats, speaker_num=4)
        return pred.speaker_diarize.postprocess(segments, labels)

    def new_path(x, sr):
        np.random.seed(0)
        return pred.speaker_diarization(x, sample_rate=sr, speaker_num=4)

    rows = []
    print(f'card: {card()}', flush=True)
    for minutes in args.minutes:
        for sr in args.rates:
            x = recording(minutes, sr, seed=int(minutes * 7 + sr % 1000))
            new_s, new_all = median_s(lambda: new_path(x, sr), args.reps)
            host_s, host_all = median_s(lambda: host_flow(x, sr), args.reps)
            equal = new_path(x, sr) == host_flow(x, sr)
            st = stage_ms(pred, x, sr)
            row = dict(minutes=minutes, sample_rate=sr, samples=int(x.size), new_s=new_s, host_s=host_s,
                       new_runs_s=new_all, host_runs_s=host_all, speedup=host_s / new_s, outputs_equal=bool(equal),
                       stages_ms=st)
            rows.append(row)
            print(json.dumps(row), flush=True)
    res = dict(card=card(), model='CAMPPlus embd_dim 192, Fbank 80, dB normalisation on, seeded random weights',
               reps=args.reps, rows=rows)
    print(f"\n{'recording':>16} {'new s':>8} {'host s':>8} {'x':>6} {'equal':>6} | {'upload':>7} {'cond':>7} {'energy':>7} "
          f"{'gather':>7} {'embed':>8} {'spectral':>8} ms  chunks")
    for r in rows:
        s = r['stages_ms']
        print(f"{r['minutes']:>5g} min {r['sample_rate'] / 1000:>5g} kHz {r['new_s']:8.3f} {r['host_s']:8.3f} {r['speedup']:6.2f} "
              f"{str(r['outputs_equal']):>6} | {s['upload']:7.1f} {s['condition']:7.1f} {s['frame_energy']:7.2f} "
              f"{s['gather_all']:7.2f} {s['embed']:8.1f} {s['spectral']:8.1f}     {s['chunks']}")
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
