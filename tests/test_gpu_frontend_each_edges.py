"""Op-level GPU tests of the ragged front-end (vp_features_each: frontend_kernel, mfcc_post_kernel and cmn_mask_kernel
with per-row lengths) at every plan branch of tests/frontend_cases.py, on the ragged cases of
tests/frontend_each_cases.py.

Each case first asserts the plan it runs (vp_frontend_plan_info == the host-plan mirror) and that the library takes
every row alone.  The call then runs on poisoned buffers: each row's tail wave[b, lens[b]:ld] holds NaN, +-inf or
3e38; feats are filled with NaNs and the scratch with NaNs, then, for a second call, with +inf; both end in a guard.
A quiet NaN alone would hide a read of an unwritten MFCC maximum (fmaxf drops NaN operands): +inf wins every maximum
and every sum, so a read of any slot no kernel wrote makes the second call differ from the first.  Row b's first T_b
frames must be bit-identical to the one-row call on its lens[b] samples and within test_gpu_frontend_edges.BARS of
the fp64 reference of that row alone (its own CMN and, for MFCC, its own top_db clamp); frames T_b .. T-1 are +0.0;
nothing past the features or the scratch is written; the scratch's row_T slot holds every T_b.

The Fbank reference takes the kernel's per-frame mean order (frontend_cases.warp_frame_mean): with torch's, the weak low
bins after DC removal move by up to 1.3e-4 log units on these rows, which is the reference's rounding, not the
kernel's.

MFCC is held to BARS['MFCC'] relative to the row's largest magnitude before CMN, the scale the kernel's fp32 rounding
follows.  On a quiet or a 2-frame row that denominator is 10 - 100 times the row's max|ref|, since CMN cancels nearly
all of the row, so there the bar is that much looser on the output itself.  The output is also held to
MFCC_ROW_REF_BAR relative to the row's own max|ref|: measured up to 2.1e-5 (a 40-frame quiet row of
test_mfcc_row_maxima_past_256) and 9.2e-6 on 2-frame rows.

Measured maxima over the ragged cases: Fbank 2.4e-6 (fbank80_1024_reflect), MelSpectrogram 1.6e-7
(mel40_200_tpc4_nocenter_pad), Spectrogram 8.3e-8 (spec1025_2048_nocache), MFCC 9.9e-7 (mfcc_many_ctas_loud_last).
Measured on an H100 80GB HBM3 (700 W); the module runs in about 13 s there."""
import ctypes as C

import numpy as np
import pytest
import torch

import frontend_cases as fc
import frontend_each_cases as ec
from mvector import _lib as L
from test_gpu_frontend_edges import BARS

pytestmark = pytest.mark.gpu

GUARD = 64                                     # floats past the end of feats and scratch
FEATS_NAN = np.uint32(0x7FC0DEAD)              # quiet NaNs with recognisable payloads
SCRATCH_NAN = np.uint32(0x7FCBAD00)
SCRATCH_INF = np.uint32(0x7F800000)            # +inf: survives fmaxf and propagates through every sum
MFCC_ROW_REF_BAR = 5e-5                        # MFCC error relative to the row's own max|ref| (measured <= 2.1e-5)


@pytest.fixture(scope='module')
def engine():
    from mvector.engine import Engine
    eng = Engine()
    yield eng
    eng.close()


def _featurizer(method, args, engine):
    from mvector.data_utils.featurizer import AudioFeaturizer
    fz = AudioFeaturizer(method, method_args=args, engine=engine)
    fz.engine                                         # configure the handle (vp_frontend_set + options)
    return fz


def _plan_info(fz, B, n):
    info = (C.c_int32 * 8)()
    rc = L.lib().vp_frontend_plan_info(fz.engine.handle, B, n, fz.feat_fun.desc.post, info)
    got = dict(zip(fc.PLAN_KEYS, list(info)))
    got['mel'] = ('plain', 'chain4')[got['mel']]
    return rc, got


def _err(method, got, ref, scale):
    """test_gpu_frontend_edges._err on one row: Fbank absolute, Mel / Spectrogram relative to the frame scale.  MFCC
    relative to the row's largest magnitude before CMN (max of ``scale``), which test_gpu_frontend_edges's max|ref|
    over a whole call of long rows is close to: a row of a few frames, or a quiet stationary one, keeps little after
    CMN, so its own max|ref| measures the cancellation, not the kernel (see the module docstring)."""
    d = np.abs(got.astype(np.float64) - ref)
    if method == 'Fbank':
        return float(d.max())
    if method == 'MFCC':
        return float(d.max() / scale.max())
    return float((d / np.maximum(scale, 1e-30)[..., None]).max())


def _poisoned(n, word):
    return torch.from_numpy(np.full(n, word, np.uint32).view(np.float32)).cuda()


def _each(fz, wave, lens, T, n, scratch_word):
    """vp_features_each on feats poisoned with FEATS_NAN and scratch with scratch_word, each with a guard.
    -> (rc, feats [B*T*F + GUARD] uint32, scratch [vp_frontend_scratch_floats(B, n) + GUARD] uint32), synchronised."""
    lib, h = L.lib(), fz.engine.handle
    B, ld = wave.shape
    nf = B * T * fz.feature_dim
    ns = int(lib.vp_frontend_scratch_floats(h, B, n))
    feats, scratch = _poisoned(nf + GUARD, FEATS_NAN), _poisoned(ns + GUARD, scratch_word)
    lens_d = torch.tensor(lens, dtype=torch.int32, device='cuda')
    rc = lib.vp_features_each(h, C.c_void_p(wave.data_ptr()), B, ld, C.c_void_p(lens_d.data_ptr()), T,
                              C.c_void_p(feats.data_ptr()), C.c_void_p(scratch.data_ptr()), fz.engine.stream_ptr())
    torch.cuda.synchronize()
    return rc, feats.cpu().numpy().view(np.uint32), scratch.cpu().numpy().view(np.uint32)


def _one_row(fz, wave, b, n):
    return fz(wave[b:b + 1, :n].contiguous()).squeeze(0).cpu().numpy()


def _check_call(fz, wave, lens, T, n, valid=None):
    """Two poisoned calls, the scratch NaN in the first and +inf in the second: their guards, row_T slots and
    padding frames, and the second bit-identical to the first.  -> feats [B, T, F] float32."""
    B = wave.shape[0]
    F = fz.feature_dim
    nf = B * T * F
    calls = []
    for word in (SCRATCH_NAN, SCRATCH_INF):
        rc, got, scr = _each(fz, wave, lens, T, n, word)
        assert rc == L.VP_OK, L.lib().vp_last_error(fz.engine.handle)
        assert (got[nf:] == FEATS_NAN).all(), 'written past the features'
        ns = scr.size - GUARD
        assert (scr[ns:] == word).all(), 'written past the scratch'
        nr = (B + 3) & ~3
        row_T = scr[ns - nr:ns].view(np.int32)
        assert row_T[:B].tolist() == [fz.num_frames(m) for m in lens]
        assert (scr[ns - nr + B:ns] == word).all()
        calls.append(got[:nf])
    assert np.array_equal(calls[1], calls[0]), 'the call reads scratch it did not write, or is not deterministic'
    feats = calls[0].view(np.float32).reshape(B, T, F)
    for b in range(B):
        tb = fz.num_frames(lens[b])
        assert not feats[b, tb:].view(np.uint32).any(), (b, 'frames past T_b are not +0.0')
        if valid is None or valid[b]:
            assert np.isfinite(feats[b, :tb]).all(), b
    return feats


def _check_row(method, args, fz, wave, feats, b, n, ref_rows=True):
    """Row b of a ragged call: bit-identical to its one-row call, within BARS of the fp64 reference of the row alone.
    -> the error measure (None when the reference is skipped)."""
    tb = fz.num_frames(n)
    one = _one_row(fz, wave, b, n)
    assert one.shape[0] == tb
    assert np.array_equal(feats[b, :tb].view(np.uint32), one.view(np.uint32)), (b, n, 'differs from one-row call')
    if not ref_rows:
        return None
    ref, scale = fc.exact_features(method, args, wave[b:b + 1, :n].cpu().numpy(), frame_mean=fc.warp_frame_mean)
    err = _err(method, feats[b:b + 1, :tb], ref, scale)
    if method == 'MFCC':
        own = float(np.abs(feats[b, :tb] - ref[0]).max() / np.abs(ref).max())
        print(f'  row {b} ({tb} frames): MFCC err {err:.3e}, relative to its own max|ref| {own:.3e}')
        assert own <= MFCC_ROW_REF_BAR, (b, n, own)
    assert err <= BARS[method], (b, n, err)
    return err


@pytest.mark.parametrize('name', ec.CASES)
def test_ragged_case(name, engine):
    """Measured maxima (H100 80GB HBM3): Fbank 2.4e-6, MelSpectrogram 1.6e-7, Spectrogram 8.3e-8, MFCC 9.9e-7."""
    c = ec.build(name)
    fz = _featurizer(c['method'], c['args'], engine)
    B = len(c['lens'])
    rc, got = _plan_info(fz, B, c['n'])
    assert rc == L.VP_OK
    plan = ec.plan_of(c)
    assert got == {k: plan[k] for k in fc.PLAN_KEYS}
    assert {k: plan[k] for k in c['intent']} == c['intent']
    for n in c['lens']:
        assert _plan_info(fz, 1, n)[0] == L.VP_OK, n           # the length mirror agrees with the library
    if c['n_min'] > 0:
        assert _plan_info(fz, 1, c['n_min'] - 1)[0] == L.VP_ERR_INVALID   # ... and so does the shortest row
    assert L.lib().vp_num_frames(fz.engine.handle, c['ld']) == c['T']
    wave = torch.from_numpy(c['wave']).cuda()
    feats = _check_call(fz, wave, c['lens'], c['T'], c['n'])
    errs = [_check_row(c['method'], c['args'], fz, wave, feats, b, n) for b, n in enumerate(c['lens'])]
    print(f'{name}: {c["method"]} err {max(errs):.3e}')


def test_mfcc_row_maxima_past_256(engine):
    """Default MFCC (n_fft 400, hop 200): one row of 4200 frames (263 tiles), quiet except for a burst in tile 259,
    between short quiet rows.  Its clamp needs the maximum of the burst, which the per-row reduction reads only past
    its first 256 maxima."""
    method, args = 'MFCC', dict()
    fz = _featurizer(method, args, engine)
    rng = np.random.default_rng(11)
    Tl = 4200
    nl = fc.lpad_for(method, args, Tl, 77)
    lens = [fc.lpad_for(method, args, t, e) for t, e in ((3, 5), (40, 0), (97, 150))]
    lens.insert(1, nl)
    ld = nl + 3
    x = np.full((len(lens), ld), np.nan, np.float32)
    for b, (n, g) in enumerate(zip(lens, (1e-2, 1e-3, 1e-4, 1e-3))):
        x[b, :n] = g * 0.1 * rng.standard_normal(n)
    f0 = 259 * 16 + 5                                   # frames f0 .. f0 + 9 of the long row
    x[1, f0 * 200:(f0 + 10) * 200] *= 3e4               # 90 dB above the rest of the row
    assert fz.num_frames(nl) == Tl and fz.num_frames(ld) == Tl
    wave = torch.from_numpy(x).cuda()
    feats = _check_call(fz, wave, lens, Tl, nl)
    for b, n in enumerate(lens):
        _check_row(method, args, fz, wave, feats, b, n)


GROUP_CONFIGS = [('Fbank', dict(sample_frequency=16000, num_mel_bins=80)), ('MFCC', dict())]


@pytest.mark.parametrize('method,args', GROUP_CONFIGS, ids=['Fbank80', 'MFCC'])
def test_group_scale(method, args, engine):
    """B = 256 rows of 0.5 - 6 s at 16 kHz, the largest evaluate group, tails poisoned with NaN: every row
    bit-identical to its one-row call, every 16th also against fp64."""
    fz = _featurizer(method, args, engine)
    rng = np.random.default_rng(12)
    lens = rng.integers(8000, 96001, 256).tolist()
    lens[100] = 96000
    ld = 96000 + 7
    x = np.full((256, ld), np.nan, np.float32)
    for b, n in enumerate(lens):
        x[b, :n] = rng.uniform(0.01, 0.5) * rng.standard_normal(n)
    wave = torch.from_numpy(x).cuda()
    T = fz.num_frames(max(lens))
    feats = _check_call(fz, wave, lens, T, max(lens))
    for b, n in enumerate(lens):
        _check_row(method, args, fz, wave, feats, b, n, ref_rows=b % 16 == 0)


CONTRACT_CONFIGS = [('Fbank', dict(num_mel_bins=80)), ('MelSpectrogram', dict(n_fft=512, hop_length=160, n_mels=64))]


@pytest.mark.parametrize('method,args', CONTRACT_CONFIGS, ids=['Fbank80', 'MelSpectrogram'])
def test_rows_the_one_row_call_refuses(method, args, engine):
    """Rows whose length a one-row call refuses (0 samples; under the Kaldi window, or within n_fft / 2 of reflect
    padding) beside valid rows, every tail NaN.  The valid rows stay exact.  A refused Kaldi row has T_b = 0 and is all
    +0.0; a refused STFT row reads nothing past its own samples, so its frames are finite."""
    fz = _featurizer(method, args, engine)
    n_min = ec.shortest_row(fz)
    rng = np.random.default_rng(13)
    lens = [0, 5000, n_min - 1, 1, 3333, n_min, 2, 4800]
    ld = 5000 + 9
    x = np.full((len(lens), ld), np.nan, np.float32)
    for b, n in enumerate(lens):
        x[b, :n] = 0.1 * rng.standard_normal(n)
    valid = [ec.length_ok(fz, n) for n in lens]
    assert valid == [False, True, False, False, True, True, False, True]
    assert [_plan_info(fz, 1, n)[0] == L.VP_OK for n in lens] == valid           # the library refuses the same rows
    wave = torch.from_numpy(x).cuda()
    T = fz.num_frames(5000)
    feats = _check_call(fz, wave, lens, T, 5000, valid=valid)
    for b, n in enumerate(lens):
        tb = fz.num_frames(n)
        if valid[b]:
            _check_row(method, args, fz, wave, feats, b, n)
        elif fz.feat_fun.desc.kind == 0:
            assert tb == 0 and not feats[b].view(np.uint32).any(), b
        else:
            assert tb >= 1 and np.isfinite(feats[b, :tb]).all(), b


def test_refusals_leave_the_features_untouched(engine):
    """null lens, T = 0, T > vp_num_frames(ld), B = 0 and an ld the length check refuses: VP_ERR_INVALID, feats
    unwritten."""
    fz = _featurizer('Fbank', dict(num_mel_bins=80), engine)
    lib, h = L.lib(), fz.engine.handle
    B, ld = 3, 4000
    T = fz.num_frames(ld)
    wave = torch.zeros(B, ld, device='cuda')
    lens = torch.tensor([4000, 400, 1000], dtype=torch.int32, device='cuda')
    feats = _poisoned(B * T * fz.feature_dim + GUARD, FEATS_NAN)
    scratch = _poisoned(int(lib.vp_frontend_scratch_floats(h, B, ld)) + GUARD, SCRATCH_NAN)
    p = [C.c_void_p(t.data_ptr()) for t in (wave, lens, feats, scratch)]
    st = fz.engine.stream_ptr()
    calls = {'null lens': (B, ld, C.c_void_p(), T), 'T = 0': (B, ld, p[1], 0), 'T > frames of ld': (B, ld, p[1], T + 1),
             'B = 0': (0, ld, p[1], T), 'ld under the window': (B, 399, p[1], 1)}
    for what, (b, n, lp, t) in calls.items():
        assert lib.vp_features_each(h, p[0], b, n, lp, t, p[2], p[3], st) == L.VP_ERR_INVALID, what
    torch.cuda.synchronize()
    assert (feats.cpu().numpy().view(np.uint32) == FEATS_NAN).all()
