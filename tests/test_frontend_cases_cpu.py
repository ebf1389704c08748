"""The front-end case table (tests/frontend_cases.py) on the CPU: its fp64 reference agrees with torchaudio and the
repository's oracles within their fp32 rounding, every case reaches the plan it names, and together the cases cover
every branch of frontend_kernel, mfcc_post_kernel and cmn_mask_kernel that the host plan can reach."""
import numpy as np
import pytest
import torch

import frontend_cases as fc
import frontend_options_oracle as ofo
from mvector import _lib as L
from oracle import frontend as ofe


def _torchaudio_features(method, args, x, ratio):
    """The reference featurizer's forward over torchaudio itself (kaldi.fbank per utterance, or the transform), CMN over
    all T frames, then the mask."""
    import torchaudio
    w = torch.from_numpy(x)
    if method == 'Fbank':
        feat = torch.stack([torchaudio.compliance.kaldi.fbank(r[None], **args) for r in w]).double()
    else:
        feat = getattr(torchaudio.transforms, method)(**args)(w).transpose(1, 2).double()
    feat = feat - feat.mean(1, keepdim=True)
    if ratio is not None:
        keep = torch.round(torch.from_numpy(ratio) * feat.shape[1]).long()
        for b, k in enumerate(keep.tolist()):
            feat[b, k:] = 0
    return feat.numpy()


def _err(method, got, ref, scale):
    """The GPU suite's metric: Fbank absolute (log units), Mel / Spectrogram relative to the frame scale, MFCC relative
    to max|ref|."""
    d = np.abs(np.asarray(got, np.float64) - ref)
    if method == 'Fbank':
        return float(d.max())
    if method == 'MFCC':
        return float(d.max() / np.abs(ref).max())
    return float((d / np.maximum(scale, 1e-30)[..., None]).max())


# fp32 rounding of the pipelines compared with: torchaudio's fp32 FFT (the Fbank log sees it at the weak low bins: up to
# 6e-4, fbank_precision_study), and the oracles, whose only difference from the reference is an fp32 log / CMN
TORCHAUDIO_BOUND = dict(Fbank=2e-3, MelSpectrogram=2e-6, Spectrogram=2e-6, MFCC=5e-5)
ORACLE_EXACT_BOUND = 5e-6         # Fbank, exact spectrum: fp32 log and CMN against fp64


@pytest.mark.parametrize('name', list(fc.CASES))
def test_reference_against_torchaudio_and_oracles(name):
    c = fc.CASES[name]
    x, ratio, keep, T = fc.materialize(name)
    ref, scale = fc.exact_features(c['method'], c['args'], x, keep)
    assert ref.shape[:2] == (x.shape[0], T)
    ta = _torchaudio_features(c['method'], c['args'], x, ratio)
    err = _err(c['method'], ta, ref, scale)
    assert err <= TORCHAUDIO_BOUND[c['method']], (name, err)
    r = None if ratio is None else torch.from_numpy(ratio)
    if c['method'] == 'Fbank':
        exact = ofo.featurize(torch.from_numpy(x), r, 'Fbank', c['args'], exact_spectrum=True).numpy()
        assert np.abs(exact - ref).max() <= ORACLE_EXACT_BOUND
        if c['args'].get('snip_edges', True):
            exact = ofe.featurize(torch.from_numpy(x), r, 'Fbank', c['args'], exact_spectrum=True).numpy()
            assert np.abs(exact - ref).max() <= ORACLE_EXACT_BOUND
    else:
        got = ofo.featurize(torch.from_numpy(x), r, c['method'], c['args']).numpy()
        assert _err(c['method'], got, ref, scale) <= TORCHAUDIO_BOUND[c['method']]
    if keep is not None:
        assert not ref[np.arange(T)[None, :] >= np.asarray(keep)[:, None]].any()


@pytest.mark.parametrize('name', list(fc.CASES))
def test_case_reaches_its_intent(name):
    c = fc.CASES[name]
    x, ratio, keep, T = fc.materialize(name)
    fz = fc.featurizer(c['method'], c['args'])
    assert fz.num_frames(x.shape[1]) == T
    if 'keep' in c:
        assert fz.keep_frames(ratio, T).tolist() == c['keep']            # the ratios round back to the intended keep
    plan = fc.plan_of(name)
    assert {k: plan[k] for k in c['intent']} == c['intent'], (name, plan)


def _facts(name):
    c = fc.CASES[name]
    x, ratio, keep, T = fc.materialize(name)
    g = fc.geometry(c['method'], c['args'])
    f = fc.featurizer(c['method'], c['args']).feat_fun
    return dict(c=c, g=g, p=fc.plan_of(name), T=T, B=x.shape[0], Lpad=x.shape[1], keep=keep or [],
                kaldi=g['kind'] == 0, pad=f.opts.pad, lens=c.get('lens', [1.0]), gain=c.get('gain'))


def _loud_last(f):
    peak = [max(np.atleast_1d(g)) for g in f['gain'] or []]
    return bool(peak) and int(np.argmax(peak)) == f['B'] - 1 and (f['B'] - 1) * f['p']['nblk'] >= 256 and \
        20 * np.log10(peak[-1] / sorted(peak)[-2]) > 80


def _one_cta_both_ends(f):
    return f['p']['tpc'] == 4 and f['p']['grid'] == 1


_STFT_MODES = {'reflect': L.FRAME_DEFAULT, 'constant': L.FRAME_STFT_CONSTANT, 'replicate': L.FRAME_STFT_REPLICATE,
               'circular': L.FRAME_STFT_CIRCULAR, 'not centred': L.FRAME_STFT_NOCENTER}

# matrix cell -> predicate over one case's facts
CELLS = {}
for _kind, _k in (('Kaldi', True), ('STFT', False)):
    for _inst in (256, 512, 1024, 2048, 0):
        CELLS[f'<{_inst}> on the {_kind} kind'] = (lambda f, k=_k, i=_inst: f['kaldi'] == k and f['p']['inst'] == i)
for _n in (480, 384, 400, 600, 200):
    CELLS[f'plan-driven n_fft {_n}'] = lambda f, n=_n: f['p']['inst'] == 0 and f['g']['N'] == n
CELLS.update({
    'plan with a radix-3 pass': lambda f: f['p']['inst'] == 0 and 3 in f['p']['radix'],
    'plan with a radix-5 pass': lambda f: f['p']['inst'] == 0 and 5 in f['p']['radix'],
    'plan with a radix-2 pass': lambda f: f['p']['inst'] == 0 and 2 in f['p']['radix'],
    'Kaldi n_fft other than 512 (frame_length / round_to_power_of_two)': lambda f: f['kaldi'] and f['g']['N'] != 512,
    'tpc 1, cache on': lambda f: f['p']['tpc'] == 1 and f['p']['cache'],
    'tpc 2, cache on': lambda f: f['p']['tpc'] == 2 and f['p']['cache'],
    'tpc 4, cache on': lambda f: f['p']['tpc'] == 4 and f['p']['cache'],
    'cache off (Spectrogram 2048, hop 512)': lambda f: not f['g']['mfcc'] and not f['p']['cache'],
    'MFCC mel stage, tpc 1': lambda f: f['g']['mfcc'] and f['p']['tpc'] == 1,
    'MFCC mel stage, tpc 2': lambda f: f['g']['mfcc'] and f['p']['tpc'] == 2,
    'MFCC mel stage, tpc 4': lambda f: f['g']['mfcc'] and f['p']['tpc'] == 4,
    'nblk % tpc != 0 (short last CTA)': lambda f: f['p']['nblk'] % f['p']['tpc'] != 0,
    'T = 1 mod 16': lambda f: f['T'] % 16 == 1 and f['T'] > 1,
    'T = 15 mod 16': lambda f: f['T'] % 16 == 15,
    'odd T (last pair has one frame)': lambda f: f['T'] % 2 == 1 and f['T'] > 1,
    'T = 1': lambda f: f['T'] == 1,
    'plain mel loop': lambda f: f['p']['mel'] == 'plain',
    'plain mel loop at 2F = G': lambda f: f['p']['inst'] != 0 and 2 * f['g']['F'] == f['p']['G'],
    '4-chain, 2F just above G (dead chains)': lambda f: f['p']['mel'] == 'chain4' and 2 * f['g']['F'] < 2 * f['p']['G'],
    '4-chain, 2F > 4G (several sweeps)': lambda f: f['p']['mel'] == 'chain4' and 2 * f['g']['F'] > 4 * f['p']['G'],
    '4-chain with vb false (odd T)': lambda f: f['p']['mel'] == 'chain4' and f['T'] % 2 == 1,
    'remove_dc, G = 32, no pre-emphasis': lambda f: f['kaldi'] and f['g']['remove_dc'] and f['p']['G'] == 32
    and f['g']['preemph'] == 0,
    'remove_dc, G = 32, pre-emphasis': lambda f: f['kaldi'] and f['g']['remove_dc'] and f['p']['G'] == 32
    and f['g']['preemph'] != 0,
    'remove_dc, G >= 64, no pre-emphasis': lambda f: f['kaldi'] and f['g']['remove_dc'] and f['p']['G'] >= 64
    and f['g']['preemph'] == 0,
    'remove_dc, G >= 64, pre-emphasis': lambda f: f['kaldi'] and f['g']['remove_dc'] and f['p']['G'] >= 64
    and f['g']['preemph'] != 0,
    'Kaldi snip_edges rows at all four 16-byte residues': lambda f: f['kaldi'] and f['g']['frame'] == L.FRAME_DEFAULT
    and f['Lpad'] % 2 == 1 and f['B'] >= 4,
    'Kaldi snip_edges=False (reflect map)': lambda f: f['kaldi'] and f['g']['frame'] == L.FRAME_KALDI_REFLECT,
    'STFT `pad` > 0 in one tpc-4 CTA': lambda f: not f['kaldi'] and f['pad'] > 0 and _one_cta_both_ends(f),
    'keep 0': lambda f: 0 in f['keep'],
    'keep 1': lambda f: 1 in f['keep'],
    'keep T - 1': lambda f: f['T'] - 1 in f['keep'],
    'keep T': lambda f: f['T'] in f['keep'],
    'keep on a 16-row boundary inside a 64-row cmn_mask CTA': lambda f: any(k % 16 == 0 and k % 64 and k < f['T']
                                                                            for k in f['keep']),
    'T > 64': lambda f: f['T'] > 64,
    'F > 128 (Spectrogram)': lambda f: f['g']['F'] > 128,
    'MFCC, B nblk > 256, loudest utterance last': lambda f: f['g']['mfcc'] and f['B'] * f['p']['nblk'] > 256
    and _loud_last(f),
    'MFCC two-stage call (vp_mfcc_mel + vp_mfcc_finish)': lambda f: f['c'] is fc.CASES[fc.TWO_STAGE]
    and f['g']['mfcc'] and _loud_last(f),
})
for _mode, _m in _STFT_MODES.items():
    CELLS[f'STFT {_mode} framing in one tpc-4 CTA across both ends'] = \
        lambda f, m=_m: not f['kaldi'] and f['g']['frame'] == m and _one_cta_both_ends(f)


def test_cases_cover_the_matrix():
    """Every cell of the matrix is reached by at least one case; prints which."""
    facts = {n: _facts(n) for n in fc.CASES}
    missing = []
    for cell, pred in CELLS.items():
        hits = [n for n, f in facts.items() if pred(f)]
        print(f'{cell}: {", ".join(hits) if hits else "-- MISSING --"}')
        if not hits:
            missing.append(cell)
    assert not missing, 'cells no case reaches: ' + '; '.join(missing)
