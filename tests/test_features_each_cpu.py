"""Host side of the ragged front-end and of the grouped evaluate / extract_features: frame counts, the ctypes binding,
the group plan and the successor rule, and the kernels' build."""
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'voiceprintrecognition-pytorch_b200', 'csrc')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')

FRAMINGS = [('Fbank', dict(sample_frequency=16000, num_mel_bins=80)),
            ('Fbank', dict(sample_frequency=16000, num_mel_bins=80, snip_edges=False)),
            ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=64)),
            ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=64, pad_mode='constant', pad=5)),
            ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=64, pad_mode='replicate')),
            ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=64, pad_mode='circular')),
            ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=64, center=False, pad=3)),
            ('Spectrogram', dict(n_fft=400, hop_length=160, normalized=True))]


def test_frame_counts_match_num_frames(tmp_path):
    """frontend_frames, the one formula behind vp_num_frames and the ragged kernels' T_b, compiled for the host, against
    AudioFeaturizer.num_frames for every framing mode."""
    if not os.path.exists(NVCC):
        pytest.skip('nvcc not installed')
    from mvector.data_utils.featurizer import AudioFeaturizer
    lens = [0, 1, 2, 159, 160, 161, 255, 256, 257, 399, 400, 401, 511, 512, 513, 16000, 16001, 160003]
    cases, want = [], []
    for method, args in FRAMINGS:
        f = AudioFeaturizer(method, method_args=args).feat_fun
        for n in lens:
            cases.append(f'{f.desc.kind} {f.opts.frame_mode} {f.win_length} {f.n_fft} {f.hop} {f.opts.pad} {n}')
            want.append(AudioFeaturizer(method, method_args=args).num_frames(n))
    src = tmp_path / 'frames.cu'
    src.write_text('#include <cstdio>\n#include "kernels.cuh"\nint main() {\n  int k, m, w, n, h, p; long long x;\n'
                   '  while (scanf("%d %d %d %d %d %d %lld", &k, &m, &w, &n, &h, &p, &x) == 7)\n'
                   '    printf("%d\\n", vpb::frontend_frames(k, m, w, n, h, p, x));\n}\n')
    exe = tmp_path / 'frames'
    r = subprocess.run([NVCC, '-std=c++17', '-I', CSRC, str(src), '-o', str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], input='\n'.join(cases) + '\n', capture_output=True, text=True, check=True).stdout
    assert [int(v) for v in out.split()] == want


def test_binding_matches_the_header():
    import ctypes as C
    from mvector import _lib as L
    hdr = open(os.path.join(ROOT, 'include', 'vpb200.h')).read()
    m = re.search(r'int vp_features_each\(([^)]*)\);', hdr)
    params = [p.strip() for p in m.group(1).split(',')]
    assert params == ['vp_handle* h', 'const float* wave', 'int32_t B', 'int32_t ld', 'const int32_t* lens', 'int32_t T',
                      'float* feats', 'float* scratch', 'void* stream']
    src = open(L.__file__).read()
    assert "'vp_features_each': (C.c_int, [vp, f32p, i32, i32, i32p, i32, f32p, f32p, vp])" in src
    assert 'vp_features_each' in L.EXPORTS


def test_group_plan():
    from mvector.trainer import plan_groups
    assert plan_groups([1] * 10, 3, 7, 1 << 30) == [(0, 6), (6, 10)]
    assert plan_groups([1] * 10, 3, 2, 1 << 30) == [(0, 3), (3, 6), (6, 9), (9, 10)]     # one slice at least
    assert plan_groups([5, 5, 5, 5, 5], 2, 256, 12) == [(0, 2), (2, 4), (4, 5)]          # the sample budget
    assert plan_groups([50, 1, 1, 1], 1, 256, 10) == [(0, 1), (1, 4)]                    # one slice past the budget
    assert plan_groups([], 3, 256, 10) == []
    # one long item never widens a group of short ones: it closes the group before it and starts a narrow one
    sizes = [10] * 8 + [1000] + [10] * 8
    assert plan_groups(sizes, 1, 256, 200) == [(0, 8), (8, 9), (9, 17)]
    assert plan_groups(sizes, 2, 256, 2500) == [(0, 8), (8, 10), (10, 17)]
    got = plan_groups(list(np.random.default_rng(0).integers(1, 100, 1000)), 8, 256, 5000)
    assert got[0][0] == 0 and got[-1][1] == 1000 and all(a[1] == b[0] for a, b in zip(got, got[1:]))
    assert all((hi - lo) % 8 == 0 and hi - lo <= 256 for lo, hi in got[:-1])
    sizes = list(np.random.default_rng(1).choice([100, 100, 100, 40000], 1000))
    for lo, hi in plan_groups(sizes, 8, 256, 1 << 16):
        assert (hi - lo) * max(sizes[lo:hi]) <= 1 << 16 or hi - lo <= 8


def test_successor_resolution_without_decoding(tmp_path, monkeypatch):
    from mvector.audio import EncodedSegment, FlacSegment, PcmSegment
    from mvector.trainer import resolve_sources
    assert resolve_sources(6, lambda j: j in (2, 4)) == [2, 2, 2, 4, 4, 2]
    assert resolve_sources(3, lambda j: False) == [None] * 3
    asked = []
    resolve_sources(5, lambda j: asked.append(j) or True)
    assert sorted(asked) == list(range(5))

    def boom(*a, **k):
        raise AssertionError('decoded')
    monkeypatch.setattr(EncodedSegment, 'decode_device', boom)
    monkeypatch.setattr(FlacSegment, '_convert', boom)
    monkeypatch.setattr(PcmSegment, '_convert', boom)
    import flac_writer as fw
    import pcm_writer as pw
    from mvector.audio import AudioSegment
    rng = np.random.default_rng(1)
    paths = []
    for i, n in enumerate([4000, 20000, 3000, 16000]):
        p = tmp_path / f'a{i}.{"flac" if i % 2 else "wav"}'
        pcm = rng.integers(-3000, 3000, n)
        p.write_bytes(fw.encode(pcm[:, None], 16000, 16) if i % 2 else pw.wav(pw.encode(pcm, 's16le'), 16000, 1, 's16le'))
        paths.append(str(p))
    src = resolve_sources(4, lambda j: AudioSegment.from_file(paths[j]).duration >= 0.5)
    assert src == [1, 1, 3, 3]


def test_frontend_builds_for_sm90a_without_spills(tmp_path):
    if not os.path.exists(NVCC):
        pytest.skip('nvcc not installed')
    r = subprocess.run([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c',
                        os.path.join(CSRC, 'frontend.cu'), '-o', str(tmp_path / 'frontend.o')],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    for k in ('frontend_kernelILi0', 'frontend_kernelILi256', 'frontend_kernelILi512', 'frontend_kernelILi1024',
              'frontend_kernelILi2048', 'mfcc_post_kernel', 'cmn_mask_kernel'):
        assert k in log
    spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert spills and all(a == '0' and b == '0' for a, b in spills), log
