"""CPU side of the conditioning and spectral edge cases (tests/stage_cases.py): every case lands on the launch path its
intent names, the tables cover each path, and the numpy restatement of the resampler's summation order stays
bit-identical to AudioSegment.resample at every rate and target of the table."""
import numpy as np
import pytest

import stage_cases as sc
from mvector.audio import AudioSegment, polyphase_taps, resample_ratio, resampled_length
from test_condition_cpu import kernel_order_gain, kernel_order_resample


@pytest.mark.parametrize('case', sc.RESAMPLE_CASES, ids=lambda c: c['name'])
def test_resample_case_reaches_its_path(case):
    assert sc.resample_ctas(case['n_in'], case['rate'], case['target']) == case['intent']


def test_resample_mirror_follows_the_tap_plan():
    """rs_filter's nt and n_pre_remove are those of the tap table the engine uploads."""
    for rate, target in {(c['rate'], c['target']) for c in sc.RESAMPLE_CASES}:
        up, down = resample_ratio(rate, target)
        if up == down:
            continue
        tab, nt, npr = polyphase_taps(up, down)
        Lh, nt_m, npr_m = sc.rs_filter(up, down)
        assert (nt_m, npr_m) == (nt, npr) and tab.size == up * nt and Lh <= up * nt


def test_resample_table_covers_every_path():
    cls = [sc.intent_class(c['intent']) for c in sc.RESAMPLE_CASES if c['target'] == 16000]
    for k in ('copy', 'staged', 'mixed', 'global'):
        assert k in cls, k
    # the down-sampling ratio at which the global-read loop starts: 224 kHz (down 14) all staged, 240 kHz (15) not
    by_rate = {c['rate']: c['intent'] for c in sc.RESAMPLE_CASES if c['target'] == 16000 and c['n_in'] == 3 * c['rate']}
    assert by_rate[224000][1] == 0 and by_rate[240000][1] > 0 and by_rate[240000][0] == 2
    assert resample_ratio(7350, 16000) == (320, 147)
    for t in (8000, 48000):
        assert any(sc.intent_class(c['intent']) != 'copy' for c in sc.RESAMPLE_CASES if c['target'] == t)
    assert any(sc.intent_class(c['intent']) == 'global' for c in sc.RESAMPLE_CASES if c['target'] == 8000)
    # n_out = 256 j - 1, 256 j, 256 j + 1 on each loop
    for rate in (44100, 240000, 384000):
        up, down = resample_ratio(rate, 16000)
        tails = {int(resampled_length(c['n_in'], up, down)) % 256
                 for c in sc.RESAMPLE_CASES if c['rate'] == rate and c['target'] == 16000 and 'nout' in c['name']}
        assert tails == {255, 0, 1}, rate
    # rows shorter than the filter half-length at a global-read rate
    up, down = resample_ratio(384000, 16000)
    short = [c['n_in'] for c in sc.RESAMPLE_CASES if c['rate'] == 384000 and c['n_in'] < 10 * max(up, down)]
    assert {1, 5, 64} <= set(short)


@pytest.mark.parametrize('rate,target', sorted({(c['rate'], c['target']) for c in sc.RESAMPLE_CASES
                                                if c['rate'] != c['target']}))
def test_kernel_order_is_bit_identical_at_every_case_rate(rate, target):
    up, down = resample_ratio(rate, target)
    rng = np.random.default_rng(rate + target)
    lengths = sorted({c['n_in'] for c in sc.RESAMPLE_CASES if (c['rate'], c['target']) == (rate, target)} | {1, 7})
    for n in lengths:
        x = (rng.standard_normal(n) * 0.1).astype(np.float32)
        seg = AudioSegment(x.copy(), rate)
        seg.resample(target)
        got = kernel_order_resample(x, up, down)
        assert got.shape == seg.samples.shape and np.array_equal(got, seg.samples), (rate, target, n)


def test_gain_cases_flag_as_their_intent():
    rows = sc.gain_rows(sc.GAIN_CASES, seed=0)
    for c, x in zip(sc.GAIN_CASES, rows):
        ref, flagged = sc.host_normalize(x, -20, c['max_gain_db'])
        assert flagged == c['flagged'], c['name']
        got, kflag = kernel_order_gain(x, -20, c['max_gain_db'])
        assert kflag == flagged, c['name']
        if not flagged:
            assert np.array_equal(np.isnan(got), np.isnan(ref)), c['name']
            ok = ~np.isnan(ref)
            assert np.array_equal(got[ok].view(np.uint32), ref[ok].view(np.uint32)), c['name']
    inf_row = rows[[c['name'] for c in sc.GAIN_CASES].index('inf_sample')]
    ref, _ = sc.host_normalize(inf_row, -20, 300.0)
    assert np.isnan(ref).sum() == 1 and np.signbit(ref[~np.isnan(ref)]).any() and not ref[~np.isnan(ref)].any()


def test_gain_table_covers_tile_edges():
    ns = {c['n'] for c in sc.GAIN_CASES}
    T = sc.GN_TILE
    assert {1, T - 1, T, T + 1, 2 * T, 3 * T + 1} <= ns
    assert any(c['flagged'] and c['max_gain_db'] == 300.0 for c in sc.GAIN_CASES)        # the 380 dB row
    assert any(c['max_gain_db'] == 10.0 and c['flagged'] for c in sc.GAIN_CASES)
    assert any(c['max_gain_db'] == 10.0 and not c['flagged'] for c in sc.GAIN_CASES)
    assert any(c['inf_at'] is not None for c in sc.GAIN_CASES)


@pytest.mark.parametrize('case', sc.SPECTRAL_CASES, ids=lambda c: c['name'])
def test_spectral_case_reaches_its_path(case):
    assert sc.spectral_plan(case['n'], case['kz']) == case['intent']


def test_spectral_table_covers_every_path():
    plans = [sc.spectral_plan(c['n'], c['kz']) for c in sc.SPECTRAL_CASES]
    assert any(p['chunks'] > 1 and p['gy'] == sc.PASS_GY_MAX for p in plans)
    assert any(p['gy'] < sc.PASS_GY_MAX for p in plans)
    assert any(p['prune_optin'] for p in plans) and any(not p['prune_optin'] for p in plans)
    # the apply_q limit at k = 16: the largest accepted n is in the table, the next one is refused
    lim = sc.apply_q_max_n(16)
    assert lim == 13656 and lim in [c['n'] for c in sc.SPECTRAL_CASES]
    assert sc.apply_q_smem(lim, 16) <= sc.OPTIN_SMEM < sc.apply_q_smem(lim + 8, 16)
    r = sc.APPLY_Q_REFUSED
    assert not sc.spectral_plan(r['n'], r['kz'])['apply_q_ok'] and sc.spectral_plan(r['n'], r['accepted_kz'])['apply_q_ok']
    # every later step of the reduction shrinks the trailing block: the passes of each case cross several grids
    for c in sc.SPECTRAL_CASES:
        gys = {sc.pass_grid(m)[1] for m in range(1, c['n'])}
        assert sc.PASS_GY_MAX in gys and len(gys) > 10


def test_tridiag_blocks():
    for n, blocks in sc.TRIDIAG_BLOCKS.items():
        assert n in [c['n'] for c in sc.SPECTRAL_CASES]
        assert sum(blocks) == n and len(set(blocks)) == 3 and set(blocks) <= set(sc.BLOCK_POOL) and min(blocks) > 16
