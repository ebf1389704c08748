"""evaluate and extract_features a group of files at a time (MVectorTrainer._group_features: one decode per codec,
one conditioning call, one vp_features_each per group) against the file-by-file loop they replaced (decode, condition
and featurize one file, one synchronising copy per file in extract_features), on seeded lists of 16 kHz mono 16-bit
WAV and FLAC files of 2-12 s.

evaluate embeds an enrolment list of --files files and a trial list of --trials files with ECAPA-TDNN and CAM++ at eval
batch size 8 (the shipped value) and 32, eval max_duration 20 s (the shipped value); extract_features writes the
features of a train list of --files files and of the two short lists.  The per-file and grouped paths alternate in one
run, --reps times each; medians are reported.  A profiled run of each path (a device synchronise around every stage,
so its total is above the timed one) splits the time into reading and parsing, decode, conditioning, front-end,
backbone (the lowering of first-seen shapes included) and, for extract_features, np.save; what is left is host glue and
the device-to-host copies.  The outputs of the two paths are compared at the timed size.

The list holds --files distinct files; their audio is drawn from --clips seeded clips (encoding 2000 FLAC files in
Python would take longer than timing them).  Card name and power limit are read in the same run.
Usage: python tools/eval_times.py [--files 2000] [--trials 200] [--reps 3] [--out file.json]"""
import argparse
import collections
import json
import os
import subprocess
import sys
import tempfile
import time
import wave

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

MODELS = {'EcapaTdnn': dict(embd_dim=192, pooling_type='ASP'), 'CAMPPlus': dict(embd_dim=192)}
FARGS = dict(sample_frequency=16000, num_mel_bins=80)


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except Exception as e:       # noqa: BLE001
        return f'unknown ({e})'


def clips(n, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = int(rng.uniform(2.0, 12.0) * 16000)
        t = np.arange(k)
        x = 6000 * np.sin(2 * np.pi * t * rng.uniform(0.005, 0.03)) + rng.normal(0, 800, k)
        out.append(np.clip(np.round(x), -32768, 32767).astype(np.int64))
    return out


def write_lists(d, fmt, n_files, n_trials, pool):
    """<d>/<fmt>_{train,enroll,trials}.txt: train and enroll the same n_files files, trials n_trials more."""
    import flac_writer as fw
    blobs = []
    for c in pool:
        if fmt == 'flac':
            blobs.append(fw.encode(c[:, None], 16000, 16, blocksize=4096,
                                   sub=lambda fi, ch, x: dict(kind='fixed', order=2)))
        else:
            blobs.append(c.astype('<i2').tobytes())
    paths = []
    for i in range(n_files + n_trials):
        p = os.path.join(d, f'{fmt}{i}.{fmt}')
        if fmt == 'flac':
            with open(p, 'wb') as f:
                f.write(blobs[i % len(blobs)])
        else:
            with wave.open(p, 'wb') as w:
                w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000)
                w.writeframes(blobs[i % len(blobs)])
        paths.append(p)
    lists = {}
    for name, sel in (('train', paths[:n_files]), ('enroll', paths[:n_files]), ('trials', paths[n_files:])):
        lists[name] = os.path.join(d, f'{fmt}_{name}.txt')
        with open(lists[name], 'w') as f:
            f.writelines(f'{p}\t{i % 100}\n' for i, p in enumerate(sel))
    return lists


def trainer(lists, model, bs):
    from mvector.trainer import MVectorTrainer
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.5, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': True, 'target_dB': -20},
                            'eval_conf': {'batch_size': bs, 'max_duration': 20}, 'train_list': lists['train'],
                            'enroll_list': lists['enroll'], 'trials_list': lists['trials']},
           'preprocess_conf': {'feature_method': 'Fbank', 'method_args': dict(FARGS)},
           'model_conf': {'model': model, 'model_args': dict(MODELS[model])}}
    return MVectorTrainer(cfg, use_gpu=True)


def per_file_extract(tr, save_dir, max_duration=100):
    """extract_features as it ran before the grouped path: successor rule, decode, condition and featurize one file,
    one copy to the host per file."""
    from mvector.audio import AudioSegment, FlacSegment
    from mvector.data_utils.featurizer import AudioFeaturizer
    pc, ds = tr.configs.preprocess_conf, tr.configs.dataset_conf.get('dataset', {})
    tr.audio_featurizer = AudioFeaturizer(feature_method=pc.feature_method, method_args=pc.get('method_args', {}))
    eng = tr.audio_featurizer.engine
    for data_list in (tr.configs.dataset_conf.train_list, tr.configs.dataset_conf.enroll_list,
                      tr.configs.dataset_conf.trials_list):
        lines = [ln for ln in open(data_list).read().splitlines() if ln.strip()]
        paths = [ln.split('\t')[0] for ln in lines]
        with open(data_list.replace('.txt', '_features.txt'), 'w') as out:
            for idx in range(len(lines)):
                j, seg = idx, None
                for _ in range(len(lines)):
                    try:
                        cand = AudioSegment.from_file(paths[j])
                        if cand.duration >= ds.get('min_duration'):
                            if isinstance(cand, FlacSegment):
                                cand.decode_device(eng)
                            seg = cand
                            break
                    except Exception:  # noqa: BLE001
                        pass
                    j = j + 1 if j < len(lines) - 1 else 0
                feature = tr.audio_featurizer(tr._condition(seg, ds.get('sample_rate'), ds.get('target_dB'), max_duration,
                                                            eng))
                feature = feature.squeeze(0).cpu().numpy()
                label = int(lines[j].split('\t')[1])
                stamp = int(time.time() * 1000)
                save_path = os.path.join(save_dir, str(label), f'{stamp}.npy')
                while os.path.exists(save_path):
                    stamp += 1
                    save_path = os.path.join(save_dir, str(label), f'{stamp}.npy')
                os.makedirs(os.path.dirname(save_path), exist_ok=True)
                np.save(save_path, feature)
                out.write(f'{save_path}\t{label}\n')


def saved(lists):
    return [np.load(ln.split('\t')[0]) for name in ('train', 'enroll', 'trials')
            for ln in open(lists[name].replace('.txt', '_features.txt')).read().splitlines()]


def timed_call(fn):
    torch.cuda.synchronize()
    s = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - s) * 1e3, r


class Stages:
    """Wall-clock per stage, a device synchronise before and after every wrapped call (profiled runs only)."""

    def __init__(self, model=None):
        from mvector import audio, flac, pcm
        from mvector.data_utils.featurizer import AudioFeaturizer
        from mvector.engine import Engine
        self.acc = collections.Counter()
        self.depth = 0
        self.sites = [(audio.AudioSegment, 'from_file', 'read_parse', True), (audio.EncodedBatch, '__init__', 'decode', False),
                      (flac.FlacBatch, 'decode_into', 'decode', False), (pcm.PcmBatch, 'decode_into', 'decode', False),
                      (Engine, 'condition', 'condition', False), (AudioFeaturizer, 'forward_each', 'frontend', False),
                      (AudioFeaturizer, '__call__', 'frontend', False), (np, 'save', 'np_save', False)]
        if model is not None:
            call_cls = next(c for c in type(model).__mro__ if '__call__' in c.__dict__)
            self.sites.append((call_cls, '__call__', 'backbone', False))
        self.saved = []

    def __enter__(self):
        for obj, name, key, cm in self.sites:
            real = obj.__dict__[name]
            self.saved.append((obj, name, real))
            fn = real.__func__ if cm else real

            def wrap(*a, _fn=fn, _key=key, **k):
                if self.depth:
                    return _fn(*a, **k)
                self.depth += 1
                torch.cuda.synchronize()
                s = time.perf_counter()
                try:
                    return _fn(*a, **k)
                finally:
                    torch.cuda.synchronize()
                    self.acc[_key] += (time.perf_counter() - s) * 1e3
                    self.depth -= 1
            setattr(obj, name, classmethod(wrap) if cm else wrap)
        return self

    def __exit__(self, *exc):
        for obj, name, real in reversed(self.saved):
            setattr(obj, name, real)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--files', type=int, default=2000)
    ap.add_argument('--trials', type=int, default=200)
    ap.add_argument('--clips', type=int, default=48)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'eval_times needs the GPU'
    from oracle import models as om
    res = {'card': card(), 'files': args.files, 'trials': args.trials, 'evaluate': [], 'extract_features': []}
    pool = clips(args.clips, 0)
    res['mean_seconds'] = round(float(np.mean([len(pool[i % len(pool)]) for i in range(args.files)])) / 16000, 3)
    with tempfile.TemporaryDirectory() as d:
        for fmt in ('wav', 'flac'):
            lists = write_lists(d, fmt, args.files, args.trials, pool)
            for model in MODELS:
                for bs in (8, 32):
                    tr = trainer(lists, model, bs)
                    tr._setup_eval()
                    tr.model.load_state_dict(om.random_state_dict(model, 80, seed=0, **MODELS[model]))
                    grouped = tr._embed_list
                    each = tr._embed_list_each
                    out = {}
                    for path, fn in (('per_file', each), ('grouped', grouped)):       # warm-up: every shape lowered
                        emb = []
                        tr._embed_list = lambda name, _fn=fn, _emb=emb: _emb.append(_fn(name)) or _emb[-1]
                        out[path] = (emb, tr.evaluate())
                    same = bool(all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
                                    for a, b in zip(out['per_file'][0], out['grouped'][0])) and
                                out['per_file'][1] == out['grouped'][1])
                    t = {'per_file': [], 'grouped': []}
                    for _ in range(args.reps):
                        for path, fn in (('per_file', each), ('grouped', grouped)):
                            tr._embed_list = fn
                            t[path].append(timed_call(tr.evaluate)[0])
                    stages = {}
                    for path, fn in (('per_file', each), ('grouped', grouped)):
                        tr._embed_list = fn
                        with Stages(tr.model) as st:
                            total = timed_call(tr.evaluate)[0]
                        stages[path] = {k: round(v, 1) for k, v in st.acc.items()}
                        stages[path]['profiled_total'] = round(total, 1)
                    row = {'format': fmt, 'model': model, 'batch_size': bs, 'equal': same,
                           'per_file_ms': round(float(np.median(t['per_file'])), 1),
                           'grouped_ms': round(float(np.median(t['grouped'])), 1), 'stages_ms': stages}
                    row['speedup'] = round(row['per_file_ms'] / row['grouped_ms'], 2)
                    print(json.dumps(row), flush=True)
                    res['evaluate'].append(row)
                    del tr
            tr = trainer(lists, 'EcapaTdnn', 8)
            t = {'per_file': [], 'grouped': []}
            outs = {}
            for rep in range(args.reps + 1):
                for path in ('per_file', 'grouped'):
                    sd = os.path.join(d, f'feat_{fmt}_{path}_{rep}')
                    fn = (lambda: per_file_extract(tr, sd)) if path == 'per_file' else \
                        (lambda: tr.extract_features(save_dir=sd))
                    ms = timed_call(fn)[0]
                    if rep == 0:
                        outs[path] = saved(lists)                       # the warm-up run is checked, not timed
                    else:
                        t[path].append(ms)
            same = len(outs['per_file']) == len(outs['grouped']) and all(
                np.array_equal(a, b) for a, b in zip(outs['per_file'], outs['grouped']))
            stages = {}
            for path in ('per_file', 'grouped'):
                sd = os.path.join(d, f'feat_{fmt}_{path}_prof')
                fn = (lambda: per_file_extract(tr, sd)) if path == 'per_file' else (lambda: tr.extract_features(save_dir=sd))
                with Stages() as st:
                    total = timed_call(fn)[0]
                stages[path] = {k: round(v, 1) for k, v in st.acc.items()}
                stages[path]['profiled_total'] = round(total, 1)
            row = {'format': fmt, 'equal': bool(same), 'rows': len(outs['grouped']),
                   'per_file_ms': round(float(np.median(t['per_file'])), 1),
                   'grouped_ms': round(float(np.median(t['grouped'])), 1), 'stages_ms': stages}
            row['speedup'] = round(row['per_file_ms'] / row['grouped_ms'], 2)
            print(json.dumps(row), flush=True)
            res['extract_features'].append(row)
    print(json.dumps({'card': res['card'], 'files': args.files, 'mean_seconds': res['mean_seconds']}))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
