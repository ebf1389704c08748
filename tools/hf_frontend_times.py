"""Cost of the HF wav2vec 2.0 front-end (vp_frontend_set_hf) at the base geometry, and of EcapaTdnn on its features.

    python tools/hf_frontend_times.py [--batch 256] [--seconds 3] [--iters 10]

Writes a seeded wav2vec2-base-shaped checkpoint (512 channels, kernels 10,3,3,3,3,2,2, strides 5,2,2,2,2,2,2, "group"
norm) to a temporary directory and, on a seeded batch of B x seconds of audio, prints:
  * the front-end's ms per batch (CUDA events, after a warm-up);
  * its ms per layer and per kernel kind (torch.profiler over one call: every slice's launches summed by position);
  * conv1's algorithmic TFLOP/s, 2 M N K over its kernel time (M = B * 4799 at 3 s, N = 512, K = 1536);
  * end-to-end EcapaTdnn (default size) embeddings per second on those features (front-end + backbone).
Prints the card's name and power limit with the numbers.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--seconds', type=float, default=3.0)
    ap.add_argument('--iters', type=int, default=10)
    a = ap.parse_args()
    sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
    import torch
    from hf_writer import write_hf_dir
    from mvector.data_utils.featurizer import AudioFeaturizer
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object
    from oracle import models as om

    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True).stdout.strip()
    except OSError:
        q = torch.cuda.get_device_name()
    B, n = a.batch, int(a.seconds * 16000)
    with tempfile.TemporaryDirectory() as td:
        write_hf_dir(td, conv_dim=(512,) * 7, seed=0)
        fz = AudioFeaturizer(feature_method=td, use_hf_model=True)
        g = torch.Generator().manual_seed(0)
        w = (torch.randn(B, n, generator=g) * 0.1).cuda()
        T = fz.num_frames(n)
        feats = torch.empty(B, T, 512, device='cuda')
        st = torch.cuda.current_stream()
        for _ in range(3):
            fz.launch(w, feats, st)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fz.launch(w, feats, st)
        e1.record()
        torch.cuda.synchronize()
        fe_ms = e0.elapsed_time(e1) / a.iters

        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fz.launch(w, feats, st)
            torch.cuda.synchronize()
        evs = [e for e in prof.events() if e.device_type.name == 'CUDA' and 'memset' not in e.name.lower()
               and 'memcpy' not in e.name.lower()]
        evs.sort(key=lambda e: e.time_range.start)
        conv_i, per_layer, per_kind = 0, [0.0] * 7, {}
        for e in evs:
            us = e.time_range.elapsed_us()
            m = re.search(r'(conv_tc\w*|hf_\w+_kernel)', e.name)
            kind = 'conv' if m and m.group(1).startswith('conv_tc') else (m.group(1) if m else e.name[:40])
            per_kind[kind] = per_kind.get(kind, 0.0) + us
            if kind == 'conv':
                per_layer[conv_i % 7] += us
                conv_i += 1
        T0 = (n - 10) // 5 + 1
        T1 = (T0 - 3) // 2 + 1
        conv1_tflops = 2.0 * B * T1 * 512 * 1536 / (per_layer[1] * 1e-6) / 1e12

        margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
        model = build_model(512, dict_to_object({'model_conf': {'model': 'EcapaTdnn', 'model_args': margs}}))
        model.load_state_dict({'0.' + k: v for k, v in om.random_state_dict('EcapaTdnn', 512, seed=0, **margs).items()})
        for _ in range(2):
            emb = model(fz(w))
        torch.cuda.synchronize()
        e0.record()
        for _ in range(a.iters):
            emb = model(fz(w))
        e1.record()
        torch.cuda.synchronize()
        e2e_ms = e0.elapsed_time(e1) / a.iters
    print(f'card: {q}')
    print(f'HF front-end, wav2vec2-base geometry, {B} x {a.seconds:g} s: {fe_ms:.2f} ms per batch')
    print('  per layer (conv kernel only, ms): ' + ', '.join(f'conv{i} {v / 1e3:.2f}' for i, v in enumerate(per_layer)))
    print('  per kernel kind (ms): ' + ', '.join(f'{k} {v / 1e3:.2f}' for k, v in sorted(per_kind.items(),
                                                                                       key=lambda kv: -kv[1])))
    print(f'  conv1 algorithmic: {conv1_tflops:.1f} TFLOP/s (M = {B * T1}, N = 512, K = 1536)')
    print(f'EcapaTdnn-on-wav2vec2 end to end: {e2e_ms:.2f} ms per batch, {B / e2e_ms * 1e3:.0f} embeddings/s '
          f'(emb {tuple(emb.shape)})')


if __name__ == '__main__':
    main()
