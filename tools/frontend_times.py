"""Front-end default path against another build of the library, and the cost of each framing option.

    python tools/frontend_times.py --base <checkout of an earlier commit, its libvpb200.so built in place>
                                   [--rounds 3] [--out DIR]

Loads the base checkout's package and library, and this tree's, in turn (one process each, VPB_LIB naming the library,
alternating for --rounds rounds) on the same seeded 256 x 3 s batch: checks that Fbank-80, MelSpectrogram-64,
Spectrogram-400 and MFCC features are bit-identical between the two, and times vp_fbank at that shape with CUDA events after a warm-up,
and beside it, through AudioFeaturizer, MelSpectrogram-64 (n_fft 1024) at 128 x 5 s and Spectrogram-400 (the mixed-radix
FFT path) at 256 x 3 s.  Then times every framing option of this tree's library at the 256 x 3 s shape.  Prints the card's
name and power limit with the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, N = 256, 48000
CONFIGS = [
    ('Fbank', dict(sample_frequency=16000, num_mel_bins=80)),
    ('MelSpectrogram', dict(sample_rate=16000, n_fft=1024, win_length=1024, hop_length=320, f_min=50.0, f_max=14000.0,
                            n_mels=64)),
    ('Spectrogram', dict()),
    ('MFCC', dict()),
]
MODES = [
    ('Fbank', dict(sample_frequency=16000, num_mel_bins=80)),
    ('Fbank', dict(sample_frequency=16000, num_mel_bins=80, snip_edges=False)),
    ('Fbank', dict(sample_frequency=16000, num_mel_bins=80, snip_edges=False, round_to_power_of_two=False)),
    ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=80)),
    ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=80, pad_mode='constant')),
    ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=80, pad_mode='replicate')),
    ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=80, pad_mode='circular')),
    ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=80, center=False, pad=40, normalized=True)),
    ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=80, norm='slaney', mel_scale='slaney')),
]


def _batch():
    import torch
    return (torch.randn(B, N, generator=torch.Generator().manual_seed(0)) * 0.1).cuda()


def _time(fn, iters=50):
    import torch
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters


def child(root, out, modes):
    import numpy as np
    import torch
    sys.path.insert(0, root)
    from loguru import logger
    logger.remove()
    from mvector import _lib as L
    from mvector.data_utils.featurizer import AudioFeaturizer
    from mvector.engine import _check
    w = _batch()
    res = {'lib': L.LIB_PATH, 'package': os.path.dirname(L.__file__)}
    feats = {}
    for method, args in CONFIGS:
        feats[method] = AudioFeaturizer(method, method_args=args)(w).cpu().numpy()
    np.savez(out + '.npz', **feats)
    fz = AudioFeaturizer('Fbank', method_args=CONFIGS[0][1])
    fz._ensure()
    h, lib = fz.engine.handle, L.lib()
    T = fz.num_frames(N)
    y = torch.empty(B, T, 80, device='cuda')
    scratch = torch.empty(int(lib.vp_frontend_scratch_floats(h, B, N)), device='cuda')
    sp = fz.engine.stream_ptr()
    res['vp_fbank_ms'] = _time(lambda: _check(h, lib.vp_fbank(h, C.c_void_p(w.data_ptr()), B, N, None,
                                                              C.c_void_p(y.data_ptr()), C.c_void_p(scratch.data_ptr()),
                                                              sp)))
    w5 = (torch.randn(128, 80000, generator=torch.Generator().manual_seed(1)) * 0.1).cuda()
    mel, spec = AudioFeaturizer('MelSpectrogram', method_args=CONFIGS[1][1]), AudioFeaturizer('Spectrogram', method_args={})
    res['beside_ms'] = {'MelSpectrogram-64 n_fft 1024, 128 x 80000': _time(lambda: mel(w5)),
                        'Spectrogram n_fft 400, 256 x 48000': _time(lambda: spec(w))}
    if modes:
        res['modes'] = []
        for method, args in MODES:
            f = AudioFeaturizer(method, method_args=args)
            res['modes'].append((method, args, _time(lambda: f(w))))
    with open(out + '.json', 'w') as fh:
        json.dump(res, fh)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--base', required=True, help='checkout to compare against, its libvpb200.so built in place')
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--child', default=None, help=argparse.SUPPRESS)
    ap.add_argument('--root', default=ROOT, help=argparse.SUPPRESS)
    ap.add_argument('--modes', action='store_true', help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        return child(a.root, a.child, a.modes)
    import numpy as np
    import torch
    roots = {'base': os.path.abspath(a.base), 'this': ROOT}
    tmp = a.out or tempfile.mkdtemp()
    os.makedirs(tmp, exist_ok=True)
    times = {k: [] for k in roots}
    beside = {k: {} for k in roots}
    modes = None
    for r in range(a.rounds):
        for k, root in roots.items():
            o = os.path.join(tmp, f'{k}{r}')
            path = os.path.join(root, 'voiceprintrecognition-pytorch_b200', 'libvpb200.so')
            cmd = [sys.executable, __file__, '--base', a.base, '--child', o, '--root', root]
            cmd += ['--modes'] if k == 'this' and r == 0 else []
            subprocess.run(cmd, check=True, env=dict(os.environ, VPB_LIB=path))
            with open(o + '.json') as fh:
                res = json.load(fh)
            assert os.path.samefile(res['lib'], path) and res['package'].startswith(root + os.sep), res
            times[k].append(res['vp_fbank_ms'])
            for name, t in res['beside_ms'].items():
                beside[k].setdefault(name, []).append(t)
            modes = res.get('modes', modes)
    fa, fb = np.load(os.path.join(tmp, 'base0.npz')), np.load(os.path.join(tmp, 'this0.npz'))
    power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True).stdout.strip()
    print(f'device: {torch.cuda.get_device_name(0)}, power limit {power}')
    for method, _ in CONFIGS:
        same = np.array_equal(fa[method], fb[method])
        print(f'{method:15s} {fa[method].shape} bit-identical: {same}')
        assert same, method
    for k in roots:
        print(f'vp_fbank {B} x {N} samples, {k:4s}: ' + ', '.join(f'{t:.3f}' for t in times[k]) + ' ms')
    for k in roots:
        for name, ts in beside[k].items():
            print(f'{name}, {k:4s}: ' + ', '.join(f'{t:.3f}' for t in ts) + ' ms')
    for method, args, t in modes:
        print(f'{t:8.3f} ms  {method} {args}')


if __name__ == '__main__':
    main()
