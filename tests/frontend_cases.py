"""Case table, host-plan mirror and fp64 reference for the op-level front-end tests (tests/test_gpu_frontend_edges.py
on the GPU, tests/test_frontend_cases_cpu.py on the CPU).

``frontend_plan`` restates csrc/frontend.cu's host plan (instantiation, FFT group size G, tiles per CTA, on-chip feature
cache, pass plan) and the kernel's mel-projection predicate, so every case can name the branch it reaches (``intent``)
and both suites can check it: the CPU suite against this mirror, the GPU suite against ``vp_frontend_plan_info`` too.

``exact_features`` is the high-precision reference of one front-end call: the framing and window pipeline in fp32 op
for op (those roundings are part of what the reference computes), the rFFT, power, `normalized` scale and mel
projection in fp64 with the featurizer's own bank, rounded to fp32 once; the log / dB as the kernel applies it; for
MFCC the call-wide maximum, top_db clamp and DCT in fp64; the CMN mean over all T frames in fp64, then the mask.
Never imported by the product."""
import numpy as np
import torch

import frontend_options_oracle as ofo
from mvector import _lib as L

FPB = 16                                          # frames per tile (api.cu FPB)
REGISTER_SIZES = (256, 512, 1024, 2048)           # frontend_kernel<N> instantiations; every other n_fft runs <0>
HALF_SM = (228 * 1024 - 2 * 1024) // 2            # frontend.cu:625
CTA_SMEM = 227 * 1024


# ---------------------------------------------------------------------------------------------------------------
# host-plan mirror (csrc/frontend.cu)
# ---------------------------------------------------------------------------------------------------------------
def frontend_group_threads(N):
    """frontend.cu:574-581."""
    first = 8 if N % 8 == 0 else 4
    G = max(32, min(256, (N // first + 31) // 32 * 32))
    while 256 % G:
        G += 32
    return G


def plan_radices(N):
    """frontend.cu:584-589: radix 8 first, then 4, 2, 5, 3."""
    n, out = N, []
    for r in (8, 4, 2, 5, 3):
        while n % r == 0 and len(out) < 12:
            out.append(r)
            n //= r
    return out


def frontend_smem_bytes(g, G, tpc, cache):
    """frontend.cu:609-615 (frontend_kernel's shared-memory carve-up)."""
    N, NG, cfr = g['N'], 256 // G, FPB * tpc
    span = (cfr - 1) * g['hop'] + g['WL']
    return (16 * (N + 8 + 2 * NG * (N + N // 8)) + 8 * ((g['mel_nw'] + 1) & ~1)
            + 4 * (((span + 3) & ~3) + ((g['WL'] + 3) & ~3) + (cfr * g['F'] if cache else 0) + 3 * g['F'] + 2 * NG + 8))


def frontend_plan(g, nblk):
    """frontend.cu:622-631 for a call of nblk 16-frame tiles per row, plus the launch shape (frontend.cu:642) and the
    kernel's mel-projection branch (frontend.cu:411: ``NFFT == 0 || 2 F <= G`` runs the plain loop, else four
    interleaved chains).  Keys as vp_frontend_plan_info's info[8]."""
    N = g['N']
    G = frontend_group_threads(N)
    radix = plan_radices(N)
    want = not g['mfcc']                          # the MFCC mel stage emits maxima, no column sums
    tpc, cache = 1, want and frontend_smem_bytes(g, G, 1, True) <= CTA_SMEM
    for t in (4, 2):
        if t <= nblk and frontend_smem_bytes(g, G, t, want) <= HALF_SM:
            tpc, cache = t, want
            break
    inst = N if N in REGISTER_SIZES else 0
    return dict(inst=inst, G=G, tpc=tpc, cache=int(cache), n_pass=len(radix),
                mel='plain' if inst == 0 or 2 * g['F'] <= G else 'chain4', nblk=nblk, grid=-(-nblk // tpc),
                radix=tuple(radix))


PLAN_KEYS = ('inst', 'G', 'tpc', 'cache', 'n_pass', 'mel', 'nblk', 'grid')     # the order of info[8]


def featurizer(method, args):
    from mvector.data_utils.featurizer import AudioFeaturizer
    return AudioFeaturizer(method, method_args=args)


def geometry(method, args):
    """What the plan reads from the configured front-end (api.cu frontend_params)."""
    f = featurizer(method, args).feat_fun
    d = f.desc
    return dict(kind=d.kind, N=d.n_fft, WL=d.win_length, hop=d.hop, F=d.n_mels, mel_nw=int(f.bank[3].size),
                mfcc=d.post == 1, remove_dc=d.remove_dc, preemph=d.preemph, frame=f.opts.frame_mode)


# ---------------------------------------------------------------------------------------------------------------
# fp64 reference
# ---------------------------------------------------------------------------------------------------------------
_NP_PAD = {L.FRAME_DEFAULT: 'reflect', L.FRAME_STFT_CONSTANT: 'constant', L.FRAME_STFT_REPLICATE: 'edge',
           L.FRAME_STFT_CIRCULAR: 'wrap'}


def dense_bank(f):
    """The featurizer's sparse bank (start, count, offset, weights) as the dense [F, n_fft/2+1] fp64 matrix the kernel
    applies (weights widened from fp32, as vp_frontend_set does)."""
    start, count, off, w = f.bank
    bank = np.zeros((len(start), f.n_fft // 2 + 1))
    for m, (s, c, o) in enumerate(zip(start, count, off)):
        bank[m, s:s + c] = w[o:o + c]
    return bank


def stft_frames(f, x):
    """torchaudio's spectrogram framing (functional.py:52-144) of x [B, L] float32: `pad` zeros at both ends, centring
    by n_fft/2 in the pad mode (none when center=False), times the window in fp32.  -> [B, T, n_fft] float32."""
    o, n = f.opts, f.n_fft
    w = np.pad(x, ((0, 0), (o.pad, o.pad))) if o.pad > 0 else x
    if o.frame_mode != L.FRAME_STFT_NOCENTER:
        w = np.pad(w, ((0, 0), (n // 2, n // 2)), mode=_NP_PAD[o.frame_mode])
    T = 1 + (w.shape[1] - n) // f.hop
    idx = np.arange(T)[:, None] * f.hop + np.arange(n)
    return w[:, idx] * f.window                                       # fp32 x fp32: one rounding, as __fmul_rn


def stft_mel(f, x):
    """Kind-1 mel stage: |rFFT|^power of the fp32 frames in fp64, times spec_scale^power, projected on the bank in fp64,
    rounded to fp32 once.  -> [B, T, F] float32."""
    z = np.fft.rfft(stft_frames(f, x).astype(np.float64), axis=-1)
    p = z.real ** 2 + z.imag ** 2
    s = f.opts.spec_scale
    p = p * (s * s) if f.desc.power == 2 else np.sqrt(p) * s
    return (p @ dense_bank(f).T).astype(np.float32)


def _log(d, s):
    """The kernel's log stage (frontend.cu emit) on fp32 values s, evaluated in fp64."""
    s = s.astype(np.float64)
    if d.use_log == 1:
        return np.log(np.maximum(s, np.float64(np.float32(d.log_floor))))
    if d.use_log == 2:
        return float(np.float32(d.db_mult)) * np.log10(np.maximum(s, np.float64(np.float32(d.log_floor))))
    if d.use_log == 3:
        return np.log(s + np.float64(np.float32(d.log_floor)))
    return s


def warp_frame_mean(frames):
    """The kernel's per-frame mean (frontend.cu, remove_dc): fp32 partial sums of the samples j = lane, lane + 32, ...
    in order, the 32 partials reduced by warp_sum's xor butterfly (common.cuh), divided by the frame length in fp32.
    After DC removal the weak low bins see little but the mean's own rounding: on tests/frontend_each_cases.py's rows,
    another rounding of the mean alone moves the reference by up to 1.3e-4 log units there.
    frames [m, size] float32 tensor -> [m, 1]."""
    f = frames.numpy()
    m, size = f.shape
    f = np.pad(f, ((0, 0), (0, -size % 32))).reshape(m, -1, 32)
    p = np.zeros((m, 32), np.float32)
    for k in range(f.shape[1]):
        p = p + f[:, k]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        p = p + p[:, lanes ^ o]
    return torch.from_numpy(p[:, :1] / np.float32(size))


def exact_features(method, args, x, keep=None, frame_mean=None):
    """One AudioFeaturizer call on x [B, Lpad] float32 -> (features [B, T, F] float64, scale [B, T]).

    ``frame_mean``: the Kaldi kind's per-frame DC offset in fp32 (None: torch's mean; warp_frame_mean: the kernel's
    summation order, which the weak low bins after DC removal are sensitive to).

    ``scale`` is what the fp32 roundings of a frame's row are proportional to: the largest magnitude before CMN in that
    frame or in the CMN means it is shifted by (for Mel / Spectrogram: the frame maximum).  ``keep`` [B] frames kept
    (None: no mask)."""
    x = np.ascontiguousarray(np.asarray(x, dtype=np.float32))
    f = featurizer(method, args).feat_fun
    d = f.desc
    if d.kind == 0:
        # kaldi.fbank: fp32 framing / DC / pre-emphasis / window, fp64 FFT, power and projection rounded to fp32 once
        mel = np.stack([ofo.kaldi_fbank(torch.from_numpy(r), exact_spectrum=True, frame_mean=frame_mean,
                                        **dict(args, use_log_fbank=False)).numpy() for r in x])
    else:
        mel = stft_mel(f, x)
    pre = _log(d, mel)
    if d.post == 1:
        if d.top_db >= 0:
            pre = np.maximum(pre, pre.max() - float(np.float32(d.top_db)))   # one maximum over the whole call
        pre = pre @ f.dct.astype(np.float64)
    mean = pre.mean(axis=1, keepdims=True)
    out = pre - mean
    scale = np.maximum(np.abs(pre).max(axis=2), np.abs(mean).max(axis=2))
    if keep is not None:
        for b, k in enumerate(keep):
            out[b, k:] = 0.0
    return out, scale


# ---------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------
def lpad_for(method, args, T, extra=0):
    """The shortest waveform that gives T frames (vp_num_frames inverted), plus `extra` < hop samples."""
    f = featurizer(method, args).feat_fun
    o, hop = f.opts, f.hop
    if f.desc.kind == 0:
        L0 = T * hop - hop // 2 if o.frame_mode == L.FRAME_KALDI_REFLECT else f.win_length + (T - 1) * hop
    elif o.frame_mode == L.FRAME_STFT_NOCENTER:
        L0 = f.n_fft + (T - 1) * hop - 2 * o.pad
    else:
        L0 = (T - 1) * hop - 2 * o.pad
    assert 0 <= extra < hop
    return L0 + extra


FB80 = dict(num_mel_bins=80)                                                   # shipped Fbank-80
FB16MS = dict(frame_length=16.0)                                               # n_fft 256
MEL256 = dict(n_fft=256, hop_length=64)

# name -> case.  T: frames; extra: samples beyond the shortest waveform with T frames (Lpad = that + extra); lens:
# per-row lengths as fractions of Lpad (rows zero-padded beyond, default all full); keep: frames kept per row (default
# round(len / Lpad * T), as predict's ratios give); gain: per-row amplitude, or a (burst, pause) pair of amplitudes that
# alternate every `segment` samples; intent: the plan the case is meant to reach.
CASES = {
    # ---- Kaldi kind (vp_fbank) ----
    'fbank80_512_tpc1_residues': dict(
        method='Fbank', args=FB80, T=47, extra=3, lens=[1.0, 1.0, 0.8, 0.55],
        intent=dict(inst=512, G=64, tpc=1, cache=1, mel='chain4'),
        why='shipped config; odd Lpad over B = 4: the rows start at all four 16-byte residues; T = 47 = 15 mod 16'),
    'fbank40_512_tpc2_nopreemph': dict(
        method='Fbank', args=dict(num_mel_bins=40, preemphasis_coefficient=0.0), T=33, extra=17, lens=[1.0, 0.7],
        intent=dict(inst=512, G=64, tpc=2, cache=1, mel='chain4'),
        why='tpc 2 with the cache, nblk 3: the last CTA owns one tile; 2F = 80 just above G = 64; G >= 64 mean, no '
            'pre-emphasis'),
    'fbank40_256_tpc4_keep': dict(
        method='Fbank', args=dict(num_mel_bins=40, frame_length=16.0, frame_shift=4.0), T=81, extra=5,
        keep=[81, 0, 1, 80, 48],
        intent=dict(inst=256, G=32, tpc=4, cache=1, mel='chain4'),
        why='<256> on the Kaldi kind, tpc 4 with the cache, nblk 6: the last CTA owns two tiles; G = 32: one warp '
            'takes both frame means; odd T on the interleaved path; keep 0 / 1 / T-1 / T and 48 (a 16-row boundary '
            'inside the first 64-row cmn_mask CTA), T > 64'),
    'fbank80_256_tpc2_sweeps': dict(
        method='Fbank', args=dict(FB16MS, num_mel_bins=80, preemphasis_coefficient=0.0), T=31, extra=100,
        lens=[1.0, 0.9, 0.4],
        intent=dict(inst=256, G=32, tpc=2, cache=1, mel='chain4'),
        why='Fbank-80 with a 16 ms window: 2F = 160 > 4G = 128 (two sweeps of the chains); G = 32 mean without '
            'pre-emphasis; T = 31 = 15 mod 16'),
    'fbank80_1024_reflect': dict(
        method='Fbank', args=dict(num_mel_bins=80, frame_length=50.0, snip_edges=False), T=17, extra=11,
        lens=[1.0, 0.75],
        intent=dict(inst=1024, G=128, tpc=1, cache=1, mel='chain4'),
        why='<1024> on the Kaldi kind, snip_edges=False (the reflect map at both ends); T = 17 = 1 mod 16'),
    'fbank80_2048_T1': dict(
        method='Fbank', args=dict(num_mel_bins=80, frame_length=100.0), T=1, extra=150, lens=[1.0, 0.97, 0.94],
        intent=dict(inst=2048, G=256, tpc=1, cache=1, mel='plain'),
        why='<2048> on the Kaldi kind, T = 1: one frame, vb false in the only pair'),
    'fbank80_400_plan': dict(
        method='Fbank', args=dict(num_mel_bins=80, round_to_power_of_two=False), T=50, extra=7,
        intent=dict(inst=0, G=64, tpc=2, cache=1, mel='plain'),
        why='plan-driven n_fft 400 = 8 2 5 5 (a radix-2 pass and two radix-5 passes) on the Kaldi kind'),
    'fbank40_480_plan': dict(
        method='Fbank', args=dict(num_mel_bins=40, frame_length=30.0, round_to_power_of_two=False), T=21, extra=0,
        intent=dict(inst=0, G=64, tpc=2, cache=1, mel='plain'),
        why='plan-driven n_fft 480 = 8 4 5 3: a radix-3 pass'),
    'fbank40_384_plan_reflect': dict(
        method='Fbank', args=dict(num_mel_bins=40, frame_length=24.0, round_to_power_of_two=False, snip_edges=False),
        T=40, extra=33,
        intent=dict(inst=0, G=64, tpc=2, cache=1, mel='plain'),
        why='plan-driven n_fft 384 = 8 8 2 3 with snip_edges=False'),
    'fbank40_600_plan_tpc4': dict(
        method='Fbank', args=dict(num_mel_bins=40, frame_length=37.5, round_to_power_of_two=False), T=79, extra=1,
        intent=dict(inst=0, G=128, tpc=4, cache=1, mel='plain'),
        why='plan-driven n_fft 600 = 8 5 5 3 at G = 128, tpc 4, nblk 5'),
    'fbank20_200_plan_g32': dict(
        method='Fbank', args=dict(num_mel_bins=20, frame_length=12.5, frame_shift=5.0, round_to_power_of_two=False),
        T=64, extra=13, lens=[1.0, 0.5],
        intent=dict(inst=0, G=32, tpc=4, cache=1, mel='plain'),
        why='plan-driven n_fft 200 = 8 5 5 at G = 32: the one-warp frame means on <0>'),
    # ---- STFT kind (vp_melspec) ----
    'mel40_256_tpc4_reflect': dict(
        method='MelSpectrogram', args=dict(MEL256, n_mels=40), T=57, extra=5,
        intent=dict(inst=256, G=32, tpc=4, cache=1, mel='chain4'),
        why='<256> on the STFT kind; T = 57 in one tpc-4 CTA whose span crosses both reflected ends'),
    'mel40_256_tpc4_constant': dict(
        method='MelSpectrogram', args=dict(MEL256, n_mels=40, pad_mode='constant'), T=57, extra=5,
        intent=dict(inst=256, G=32, tpc=4, cache=1, mel='chain4'), why='zero-padded ends in one tpc-4 CTA'),
    'mel40_256_tpc4_replicate': dict(
        method='MelSpectrogram', args=dict(MEL256, n_mels=40, pad_mode='replicate'), T=57, extra=5,
        intent=dict(inst=256, G=32, tpc=4, cache=1, mel='chain4'), why='replicated ends in one tpc-4 CTA'),
    'mel40_200_tpc4_circular': dict(
        method='MelSpectrogram', args=dict(n_fft=200, hop_length=50, n_mels=40, pad_mode='circular'), T=63, extra=9,
        intent=dict(inst=0, G=32, tpc=4, cache=1, mel='plain'),
        why='plan-driven n_fft 200 on the STFT kind; wrapped ends in one tpc-4 CTA'),
    'mel40_200_tpc4_nocenter_pad': dict(
        method='MelSpectrogram', args=dict(n_fft=200, hop_length=50, n_mels=40, center=False, pad=37), T=55, extra=3,
        intent=dict(inst=0, G=32, tpc=4, cache=1, mel='plain'),
        why='center=False with `pad` zeros: the span crosses both ends of the signal into the pad'),
    'mel40_256_tpc4_pad_normalized': dict(
        method='MelSpectrogram', args=dict(MEL256, n_mels=40, pad=50, normalized=True), T=61, extra=2,
        intent=dict(inst=256, G=32, tpc=4, cache=1, mel='chain4'),
        why='`pad` zeros inside the reflect centring, normalized by the window norm'),
    'mel16_256_plain_at_G': dict(
        method='MelSpectrogram', args=dict(MEL256, n_mels=16), T=35, extra=1, lens=[1.0, 0.6],
        intent=dict(inst=256, G=32, tpc=2, cache=1, mel='plain'),
        why='the plain mel loop at 2F = G = 32 on a register-resident kernel; odd T'),
    'mel17_256_chain_dead': dict(
        method='MelSpectrogram', args=dict(MEL256, n_mels=17, power=1.0, normalized='frame_length', f_min=300.0),
        T=33, extra=0,
        intent=dict(inst=256, G=32, tpc=2, cache=1, mel='chain4'),
        why='2F = 34 just above G = 32: three of the four chains dead for most threads; |X| scaled by 1/sqrt(n_fft)'),
    'mel64_512_chain': dict(
        method='MelSpectrogram', args=dict(n_fft=512, hop_length=160, n_mels=64), T=30, extra=99,
        intent=dict(inst=512, G=64, tpc=1, cache=1, mel='chain4'),
        why='<512> on the STFT kind'),
    'mel64_1024_plain_at_G': dict(
        method='MelSpectrogram', args=dict(n_fft=1024, hop_length=320, n_mels=64, f_min=50.0, f_max=7000.0), T=15,
        extra=0, intent=dict(inst=1024, G=128, tpc=1, cache=1, mel='plain'),
        why='<1024> on the STFT kind: the plain loop at 2F = G = 128'),
    'mel128_400_plan': dict(
        method='MelSpectrogram', args=dict(hop_length=160), T=49, extra=5, lens=[1.0, 0.3],
        intent=dict(inst=0, G=64, tpc=2, cache=1, mel='plain'),
        why='torchaudio default n_fft 400 (8 2 5 5), 128 mel bins, plan-driven'),
    'mel40_480_plan': dict(
        method='MelSpectrogram', args=dict(n_fft=480, hop_length=120, n_mels=40, norm='slaney', mel_scale='slaney'),
        T=18, extra=1,
        intent=dict(inst=0, G=64, tpc=2, cache=1, mel='plain'), why='plan-driven n_fft 480 = 8 4 5 3'),
    'mel40_384_plan': dict(
        method='MelSpectrogram', args=dict(n_fft=384, hop_length=96, n_mels=40), T=66, extra=7,
        intent=dict(inst=0, G=64, tpc=4, cache=1, mel='plain'), why='plan-driven n_fft 384 = 8 8 2 3, tpc 4'),
    'mel40_600_plan': dict(
        method='MelSpectrogram', args=dict(n_fft=600, hop_length=150, n_mels=40), T=16, extra=149,
        intent=dict(inst=0, G=128, tpc=1, cache=1, mel='plain'), why='plan-driven n_fft 600 = 8 5 5 3; T = 16'),
    'spec1025_2048_nocache': dict(
        method='Spectrogram', args=dict(n_fft=2048, hop_length=512), T=20, extra=100, lens=[1.0, 0.5],
        intent=dict(inst=2048, G=256, tpc=1, cache=0, mel='chain4'),
        why='<2048> on the STFT kind; F = 1025: no on-chip cache (the CMN sums reread the features), 2F > 4G: '
            'three sweeps of the chains, F > 128 columns in cmn_mask'),
    'spec129_256_tpc2': dict(
        method='Spectrogram', args=dict(n_fft=256, hop_length=64), T=45, extra=3,
        intent=dict(inst=256, G=32, tpc=2, cache=1, mel='chain4'), why='F = 129 > 128 with the cache, tpc 2'),
    # ---- MFCC (vp_mfcc: the mel stage emits per-CTA maxima) ----
    'mfcc_1024_tpc1': dict(
        method='MFCC', args=dict(melkwargs=dict(n_fft=1024, hop_length=256, n_mels=128)), T=31, extra=0,
        lens=[1.0, 0.6], intent=dict(inst=1024, G=128, tpc=1, cache=0, mel='chain4'),
        why='MFCC mel stage at tpc 1'),
    'mfcc_400_tpc2': dict(
        method='MFCC', args=dict(), T=47, extra=11, lens=[1.0, 0.5, 0.25],
        intent=dict(inst=0, G=64, tpc=2, cache=0, mel='plain'),
        why='the default MFCC (n_fft 400) mel stage at tpc 2, nblk 3'),
    'mfcc_256_tpc4': dict(
        method='MFCC', args=dict(n_mfcc=20, melkwargs=dict(MEL256, n_mels=32)), T=77, extra=30,
        intent=dict(inst=256, G=32, tpc=4, cache=0, mel='chain4'),
        why='MFCC mel stage at tpc 4, nblk 5'),
    'mfcc_many_ctas_loud_last': dict(
        method='MFCC', args=dict(), T=250, extra=0, lens=[1.0] * 20, gain=[1e-3] * 19 + [(30.0, 3e-4)],
        segment=4000, intent=dict(inst=0, G=64, tpc=2, cache=0, mel='plain'),
        why='B nblk = 20 x 16 = 320 > 256 per-CTA maxima, the loudest utterance last (its maxima at index >= 304): '
            'the strided reductions must read past their first sweep; the quiet rows and the loud row\'s pauses sit '
            '> 80 dB below its bursts, so the top_db clamp holds most frames, and the bursts give the CMN output a '
            'spread of the size of the dB values themselves'),
}
TWO_STAGE = 'mfcc_many_ctas_loud_last'            # also run as vp_mfcc_mel + vp_mfcc_finish


def materialize(name):
    """-> (x [B, Lpad] float32, ratio [B] float32 or None, keep [B] list or None, T)."""
    c = CASES[name]
    Lpad = lpad_for(c['method'], c['args'], c['T'], c.get('extra', 0))
    lens = [int(round(fr * Lpad)) for fr in c.get('lens', [1.0])]
    B = len(c['keep']) if 'keep' in c else len(lens)
    lens = (lens * B)[:B] if len(lens) == 1 else lens
    gain = c.get('gain', [1.0] * B)
    rng = np.random.default_rng(sum(map(ord, name)))
    x = np.zeros((B, Lpad), np.float32)
    for b in range(B):
        g = np.resize(np.repeat(gain[b], c.get('segment', 1)), lens[b])     # a pair alternates every `segment` samples
        x[b, :lens[b]] = g * 0.1 * rng.standard_normal(lens[b])
    T = c['T']
    if 'keep' in c:
        ratio = np.asarray(c['keep'], np.float64) / T
    elif any(n != Lpad for n in lens):
        ratio = np.asarray(lens, np.float64) / Lpad
    else:
        return x, None, None, T
    ratio = ratio.astype(np.float32)
    keep = [int(k) for k in torch.round(torch.from_numpy(ratio) * T).to(torch.int32)]   # featurizer keep_frames
    return x, ratio, keep, T


def plan_of(name):
    c = CASES[name]
    return frontend_plan(geometry(c['method'], c['args']), -(-c['T'] // FPB))
