"""Host side of the device input conditioning (csrc/condition.cu): the tap plan against scipy's resample_poly recipe, a
numpy restatement of the kernel's summation order against AudioSegment.resample, the gain arithmetic against
AudioSegment.normalize, and the sm_90a build of the new kernels."""
import os
import re
import subprocess

import numpy as np
import pytest
from scipy.signal import firwin

from mvector.audio import AudioSegment, polyphase_taps, resample_ratio, resampled_length

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RATES = (8000, 11025, 12000, 22050, 24000, 32000, 44100, 48000, 96000)


def kernel_order_resample(x, up, down):
    """vp_resample's arithmetic in numpy: output j = upfirdn output i = j + n_pre_remove, summed over k in increasing
    order from 0.0, every product and sum rounded on its own, taps read from the per-phase table."""
    tab, nt, n_pre_remove = polyphase_taps(up, down)
    max_rate = max(up, down)
    half_len = 10 * max_rate
    Lh = down - half_len % down + 2 * half_len + 1
    xd = np.asarray(x, dtype=np.float32).astype(np.float64)
    n_in = xd.size
    n_out = int(resampled_length(n_in, up, down))
    i = np.arange(n_pre_remove, n_pre_remove + n_out, dtype=np.int64)
    t0 = i * down
    q, p = t0 // up, t0 % up
    kmax = np.minimum(q, n_in - 1)
    kmin = np.maximum(-(-(t0 - (Lh - 1)) // up), 0)
    acc = np.zeros(n_out)
    for t in range(int((kmax - kmin + 1).max()) if n_out else 0):
        k = kmin + t
        ok = k <= kmax
        prod = xd[np.clip(k, 0, n_in - 1)] * tab[np.clip(p * nt + (q - k), 0, tab.size - 1)]
        acc = np.where(ok, acc + prod, acc)
    return acc.astype(np.float32)


def kernel_order_gain(x, target_db, max_gain_db=300.0, tile=4096):
    """vp_gain_normalize's arithmetic: per-tile sums of the squares combined in tile order, then the float64 factor and
    (float)(x * factor).  -> (row, flagged)."""
    xd = np.asarray(x, dtype=np.float32).astype(np.float64)
    s = 0.0
    for t in range(0, xd.size, tile):
        s += float(np.sum(xd[t:t + tile] ** 2))
    with np.errstate(divide='ignore', invalid='ignore'):
        gain = target_db - 10.0 * np.log10(s / xd.size)
    if gain > max_gain_db:
        return np.asarray(x, dtype=np.float32), True
    return (xd * (10.0 ** (gain / 20.0))).astype(np.float32), False


@pytest.mark.parametrize('sr', RATES)
def test_tap_plan_follows_scipy_recipe(sr):
    up, down = resample_ratio(sr, 16000)
    assert np.gcd(up, down) == 1 and up * sr == down * 16000
    tab, nt, n_pre_remove = polyphase_taps(up, down)
    max_rate = max(up, down)
    half_len = 10 * max_rate
    h = firwin(2 * half_len + 1, 1.0 / max_rate, window=('kaiser', 5.0)) * up
    n_pre_pad = down - half_len % down
    assert n_pre_remove == (half_len + n_pre_pad) // down
    hpad = np.concatenate([np.zeros(n_pre_pad), h])
    assert nt == -(-hpad.size // up) and tab.size == up * nt
    p, m = np.divmod(np.arange(tab.size), nt)
    src = p + m * up
    inside = src < hpad.size
    assert np.array_equal(tab[inside], hpad[src[inside]]) and not tab[~inside].any()
    for n in (1, 17, 1000, sr * 3 + 7):
        seg = AudioSegment(np.ones(n, dtype=np.float32), sr)
        seg.resample(16000)
        assert seg.samples.size == int(resampled_length(n, up, down))


def test_resampled_length_is_int64():
    # ten minutes at 44.1 kHz times up = 160 overflows int32
    n = 44100 * 600
    assert int(resampled_length(np.int32(n), np.int32(160), np.int32(441))) == -(-n * 160 // 441) == 9600000


@pytest.mark.parametrize('sr', RATES)
def test_kernel_order_is_bit_identical_to_resample_poly(sr):
    rng = np.random.default_rng(sr)
    up, down = resample_ratio(sr, 16000)
    half_len = 10 * max(up, down)
    lengths = [1, 5, min(half_len // 2, 3000), 1000, sr * 3 + 7] + [int(v) for v in rng.integers(sr // 4, sr, 3)]
    for n in lengths:
        x = (rng.standard_normal(n) * 0.1).astype(np.float32)
        seg = AudioSegment(x.copy(), sr)
        seg.resample(16000)
        got = kernel_order_resample(x, up, down)
        assert got.shape == seg.samples.shape and np.array_equal(got, seg.samples), (sr, n)


def test_gain_arithmetic_matches_normalize():
    rng = np.random.default_rng(7)
    for n in (1, 400, 4096, 4097, 48000, 50001):
        x = (rng.standard_normal(n) * rng.uniform(0.001, 0.5)).astype(np.float32)
        seg = AudioSegment(x.copy(), 16000)
        seg.normalize(target_db=-20)
        got, flagged = kernel_order_gain(x, -20)
        assert not flagged and np.array_equal(got, seg.samples), n


def test_silent_row_is_flagged_and_raises():
    x = np.zeros(16000, dtype=np.float32)
    got, flagged = kernel_order_gain(x, -20)
    assert flagged and not got.any()
    with pytest.raises(ValueError):
        AudioSegment(x, 16000).normalize(target_db=-20)


def test_condition_kernels_build_for_sm90a_without_spills(tmp_path):
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    if not os.path.exists(nvcc):
        pytest.skip('nvcc not installed')
    src = os.path.join(ROOT, 'voiceprintrecognition-pytorch_b200', 'csrc', 'condition.cu')
    r = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '-Xptxas', '-v', '-c', src,
                        '-o', str(tmp_path / 'condition.o')], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    for k in ('resample_kernel', 'gain_energy_kernel', 'gain_factor_kernel', 'gain_apply_kernel'):
        assert k in log
    spills = re.findall(r'(\d+) bytes spill stores, (\d+) bytes spill loads', log)
    assert spills and all(a == '0' and b == '0' for a, b in spills), log
