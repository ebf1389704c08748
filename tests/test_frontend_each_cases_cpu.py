"""The ragged case table (tests/frontend_each_cases.py) on the CPU: every case runs the plan its source case names, every
row is a length a one-row call accepts, and together the cases reach every ragged edge of frontend_kernel,
mfcc_post_kernel and cmn_mask_kernel that the GPU suite checks."""
import numpy as np
import pytest
import torch

import frontend_cases as fc
import frontend_each_cases as ec
from mvector import _lib as L


@pytest.fixture(scope='module')
def built():
    return {n: ec.build(n) for n in ec.CASES}


@pytest.mark.parametrize('name', ec.CASES)
def test_case_reaches_its_intent(name, built):
    c = built[name]
    fz = fc.featurizer(c['method'], c['args'])
    plan = ec.plan_of(c)
    assert {k: plan[k] for k in c['intent']} == c['intent'], (name, plan)
    assert fz.num_frames(c['n']) == c['T'] == fz.num_frames(c['ld'])
    assert fz.num_frames(c['Lmax']) == fc.CASES[name]['T'] == c['Tb'][c['longest']]
    assert max(c['lens']) == c['Lmax'] and 0 < c['longest'] < len(c['lens']) - 1
    assert (c['ld'] - c['Lmax']) % 2 == 1
    assert c['T'] > max(c['Tb']) if c['wide'] else c['T'] == max(c['Tb'])
    for b, n in enumerate(c['lens']):
        assert ec.length_ok(fz, n), (b, n)                       # the length mirror accepts every row
        assert c['Tb'][b] == fz.num_frames(n)
        tail = c['wave'][b, n:]
        assert tail.size and np.array_equal(tail, np.full_like(tail, c['poison']), equal_nan=True)
        assert np.isfinite(c['wave'][b, :n]).all()
    assert c['n_min'] == 0 or not ec.length_ok(fz, c['n_min'] - 1)   # the shortest row is the shortest accepted


def test_length_mirror_matches_the_rules():
    """length_ok on hand-worked lengths: the Kaldi window, reflect n_fft/2 < L + 2 pad, circular <=, center=False
    n_fft <= L + 2 pad, and a non-empty signal for constant / replicate."""
    def fz(method, args):
        return fc.featurizer(method, args)
    k = fz('Fbank', dict(num_mel_bins=80))
    assert not ec.length_ok(k, 399) and ec.length_ok(k, 400) and ec.shortest_row(k) == 400
    r = fz('MelSpectrogram', dict(n_fft=512, hop_length=160))
    assert not ec.length_ok(r, 256) and ec.length_ok(r, 257)
    rp = fz('MelSpectrogram', dict(n_fft=512, hop_length=160, pad=5))
    assert not ec.length_ok(rp, 246) and ec.length_ok(rp, 247)
    c = fz('MelSpectrogram', dict(n_fft=512, hop_length=160, pad_mode='circular'))
    assert not ec.length_ok(c, 255) and ec.length_ok(c, 256)
    n = fz('MelSpectrogram', dict(n_fft=512, hop_length=160, center=False, pad=3))
    assert not ec.length_ok(n, 505) and ec.length_ok(n, 506)
    for mode in ('constant', 'replicate'):
        z = fz('MelSpectrogram', dict(n_fft=512, hop_length=160, pad_mode=mode))
        assert not ec.length_ok(z, 0) and ec.length_ok(z, 1)


def _facts(c):
    g = fc.geometry(c['method'], c['args'])
    p = ec.plan_of(c)
    f = fc.featurizer(c['method'], c['args']).feat_fun
    tb = np.asarray(c['Tb'])
    nb = -(-tb // fc.FPB)
    return dict(c=c, g=g, p=p, kaldi=g['kind'] == 0, tb=tb, nb=nb, T=c['T'], B=len(tb), hop=f.hop,
                lens=np.asarray(c['lens']))


def _dead_in_cta(f):
    """tpc > 1: a row's last live tile shares its CTA with a dead tile of the grid (nb % tpc != 0 and tile nb exists,
    nb < the call's nblk).  tpc 1: a row ends inside a tile and the grid goes on past it."""
    t, inside = f['p']['tpc'], f['nb'] < f['p']['nblk']
    if t == 1:
        return bool((inside & (f['tb'] % fc.FPB != 0)).any())
    return bool((inside & (f['nb'] % t != 0)).any())


def _segment_rms(x, n, seg):
    """RMS of x[:n] over consecutive segments of seg samples."""
    k = -(-n // seg)
    s = np.pad(x[:n].astype(np.float64), (0, k * seg - n)).reshape(k, seg)
    cnt = np.minimum(seg, n - seg * np.arange(k))
    return np.sqrt((s * s).sum(1) / cnt)


def _mfcc_gains(f):
    """In the built waves: a loud row whose bursts sit > 80 dB above its pauses, and a quiet row whose loudest
    segment sits > 80 dB below the call's loudest, so the whole call's top_db clamp would take all of it and its own
    clamp does not."""
    if not f['g']['mfcc']:
        return False
    seg = 8 * f['hop']                                              # the burst / pause period of build()
    rms = [_segment_rms(f['c']['wave'][b], n, seg) for b, n in enumerate(f['lens'])]
    peak = max(r.max() for r in rms)
    loud = any(r.max() > 1e4 * r.min() for r in rms)
    quiet = any(r.max() * 1e4 < peak for r in rms)
    return loud and quiet


_MODES = {'Kaldi snip_edges': (True, L.FRAME_DEFAULT), 'Kaldi reflect': (True, L.FRAME_KALDI_REFLECT),
          'STFT reflect': (False, L.FRAME_DEFAULT), 'STFT constant': (False, L.FRAME_STFT_CONSTANT),
          'STFT replicate': (False, L.FRAME_STFT_REPLICATE), 'STFT circular': (False, L.FRAME_STFT_CIRCULAR),
          'STFT not centred': (False, L.FRAME_STFT_NOCENTER)}

CELLS = {}
CELLS['tpc 1: a row ends inside a tile, the grid goes on past it'] = lambda f: f['p']['tpc'] == 1 and _dead_in_cta(f)
for _t in (2, 4):
    CELLS[f'tpc {_t}: a row\'s last live tile in a CTA with a dead tile of the grid'] = \
        lambda f, t=_t: f['p']['tpc'] == t and _dead_in_cta(f)
for _kind, _k in (('Kaldi', True), ('STFT', False)):
    CELLS[f'{_kind} kind'] = lambda f, k=_k: f['kaldi'] == k
for _mode, (_k, _m) in _MODES.items():
    CELLS[f'{_mode} framing'] = lambda f, k=_k, m=_m: f['kaldi'] == k and f['g']['frame'] == m
for _inst in (0, 256, 512, 1024, 2048):
    CELLS[f'inst {_inst}'] = lambda f, i=_inst: f['p']['inst'] == i
CELLS.update({
    'cache on': lambda f: f['p']['cache'] == 1,
    'cache off, Fbank / Mel / Spectrogram (CMN sums reread the features)': lambda f: not f['p']['cache']
    and not f['g']['mfcc'],
    'cache off, MFCC': lambda f: not f['p']['cache'] and f['g']['mfcc'],
    'T > T_b for every row (stride past the longest row)': lambda f: (f['tb'] < f['T']).all(),
    'T > T_b for every row, STFT constant': lambda f: (f['tb'] < f['T']).all() and not f['kaldi']
    and f['g']['frame'] == L.FRAME_STFT_CONSTANT,
    'T > T_b for every row, STFT not centred': lambda f: (f['tb'] < f['T']).all()
    and f['g']['frame'] == L.FRAME_STFT_NOCENTER,
    'T > T_b for every row, Kaldi': lambda f: (f['tb'] < f['T']).all() and f['kaldi'],
    'T > T_b for every row, MFCC': lambda f: (f['tb'] < f['T']).all() and f['g']['mfcc'],
    'odd ld - Lmax': lambda f: (f['c']['ld'] - f['c']['Lmax']) % 2 == 1,
    'rows at all four 16-byte residues': lambda f: f['c']['ld'] % 2 == 1 and f['B'] >= 4,
    'shortest row of the Kaldi kind: one frame': lambda f: f['kaldi'] and f['g']['frame'] == L.FRAME_DEFAULT
    and f['tb'][0] == 1,
    'shortest row of centred STFT: more than one frame': lambda f: not f['kaldi']
    and f['g']['frame'] != L.FRAME_STFT_NOCENTER and f['tb'][0] > 1,
    'T_b = 15 mod 16': lambda f: (f['tb'] % 16 == 15).any(),
    'T_b = 0 mod 16, below T': lambda f: ((f['tb'] % 16 == 0) & (f['tb'] < f['T'])).any(),
    'T_b = 1 mod 16, above 1': lambda f: ((f['tb'] % 16 == 1) & (f['tb'] > 1)).any(),
    'T_b = 16 tpc - 1, tpc > 1': lambda f: f['p']['tpc'] > 1 and (f['tb'] == 16 * f['p']['tpc'] - 1).any(),
    'T_b = 16 tpc + 1, tpc > 1': lambda f: f['p']['tpc'] > 1 and (f['tb'] == 16 * f['p']['tpc'] + 1).any(),
    'T_b = T - 1': lambda f: (f['tb'] == f['T'] - 1).any(),
    'a row off the hop grid': lambda f: (f['lens'] % f['hop'] != 0).any(),
    'longest row neither first nor last': lambda f: 0 < int(np.argmax(f['lens'])) < f['B'] - 1,
    'MFCC: a quiet row and a loud row with bursts > 80 dB above its pauses': _mfcc_gains,
})
for _p in ec.POISONS:
    CELLS[f'tail poison {_p}'] = lambda f, v=_p: np.array_equal(np.float32(f['c']['poison']), np.float32(v),
                                                                 equal_nan=True)


def test_cases_cover_the_matrix(built):
    """Every ragged edge is reached by at least one case; prints which."""
    facts = {n: _facts(c) for n, c in built.items()}
    missing = []
    for cell, pred in CELLS.items():
        hits = [n for n, f in facts.items() if pred(f)]
        print(f'{cell}: {", ".join(hits) if hits else "-- MISSING --"}')
        if not hits:
            missing.append(cell)
    assert not missing, 'cells no case reaches: ' + '; '.join(missing)


@pytest.mark.parametrize('size', [400, 256, 1600, 384, 200, 37, 32, 1])
def test_warp_frame_mean_is_a_mean(size):
    """frontend_cases.warp_frame_mean (the kernel's summation order) agrees with the fp64 mean within the fp32 bound of
    its ceil(size / 32) sequential and 5 butterfly additions, and with torch's mean within a few ulps of the mean."""
    rng = np.random.default_rng(size)
    x = (0.3 + 0.1 * rng.standard_normal((200, size))).astype(np.float32)
    got = fc.warp_frame_mean(torch.from_numpy(x)).numpy()[:, 0].astype(np.float64)
    m64 = x.astype(np.float64).mean(1)
    bound = (-(-size // 32) + 6) * 2.0 ** -24 * np.abs(x).astype(np.float64).mean(1)
    assert (np.abs(got - m64) <= bound).all()
    ulp = np.spacing(np.abs(x.mean(1)))
    tm = torch.from_numpy(x).mean(1).numpy().astype(np.float64)
    assert (np.abs(got - tm) <= 4 * ulp).all(), np.abs(got - tm).max() / ulp.max()
    if size == 1:
        assert np.array_equal(got, x[:, 0])
