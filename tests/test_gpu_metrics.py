"""Device verification metrics (csrc/verify.cu through vp_verify_metrics / Engine.verification_metrics) against the numpy
restatement (oracle/metrics.py), the host metric functions with a stable sort, and the reference's evaluate golden."""
import os
import wave

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import metrics as om

pytestmark = pytest.mark.gpu

TILE = 4096
FIELDS = ('n_target', 'n_impostor', 'x1', 'x2', 'target_x1', 'impostor_x1', 'target_x2', 'impostor_x2', 'min_cost',
          'argmin')


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    e = Engine()
    yield e
    e.close()


def _scores(kind, n, seed):
    rng = np.random.RandomState(seed)
    if kind == 'ties':                                   # few distinct values, labels alternate inside every group
        s = np.round(rng.rand(n) * 40).astype(np.float32) / np.float32(8)
        lab = (np.arange(n) % 2).astype(np.int32)
    elif kind == 'equal':
        s = np.full(n, 0.25, dtype=np.float32)
        lab = (rng.rand(n) < 0.5).astype(np.int32)
    elif kind == 'special':
        pool = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-45, -1e-45, 0.5, -0.5], dtype=np.float32)
        s = np.where(rng.rand(n) < 0.5, pool[rng.randint(0, len(pool), n)], rng.randn(n).astype(np.float32))
        s = s.astype(np.float32)
        lab = rng.randint(0, 2, n).astype(np.int32)
    else:
        s = rng.randn(n).astype(np.float32)
        lab = (rng.rand(n) < 0.1).astype(np.int32)
    return s, lab


def _same_result(got, want):
    for f in FIELDS:
        assert getattr(got, f) == getattr(want, f), (f, getattr(got, f), getattr(want, f))
    assert (np.isnan(got.threshold) and np.isnan(want.threshold)) or got.threshold == want.threshold


@pytest.mark.parametrize('n,kind', [(1, 'ties'), (TILE - 1, 'ties'), (TILE, 'ties'), (TILE + 1, 'ties'),
                                    (3 * TILE + 7, 'ties'), (3 * TILE + 7, 'equal'), (3 * TILE + 7, 'special'),
                                    ((1 << 20) + 3, 'ties'), ((1 << 20) + 3, 'special'), ((1 << 20) + 3, 'equal'),
                                    ((1 << 26) + 5, 'ties')])
def test_sort_is_numpy_stable_argsort(eng, n, kind):
    s, lab = _scores(kind, n, seed=n % 1000)
    res, ss, sl = eng.verify(s, labels=lab, sorted_out=True)
    keys, codes = om.stable_sort(s, lab)
    assert np.array_equal(om.score_keys(ss.cpu().numpy()), keys)
    assert np.array_equal(sl.cpu().numpy(), codes)
    _same_result(res, om.verify(s, lab)[0])


@pytest.mark.parametrize('kind', ['plain', 'ties'])
@pytest.mark.parametrize('params', [(0.01, 1, 1), (0.05, 10, 1), (0.3, 1, 3.5)])
def test_flat_metrics_bit_identical_to_oracle(eng, kind, params):
    from mvector.metric.verification import metrics_from_result
    p, cm, cf = params
    for n in (5000, 3 * TILE + 7, 200003):
        s, lab = _scores(kind, n, seed=n)
        if kind == 'ties':
            lab = (np.random.RandomState(n).rand(n) < 0.2).astype(np.int32)
        res = eng.verify(s, labels=lab, p_target=p, c_miss=cm, c_fa=cf)[0]
        want = om.verify(s, lab, p, cm, cf)[0]
        _same_result(res, want)
        assert eng.verification_metrics(torch.from_numpy(s).cuda(), labels=lab, p_target=p, c_miss=cm, c_fa=cf) == \
            metrics_from_result(want, p, cm, cf)


@pytest.mark.parametrize('nt,ne', [(37, 113), (301, 97), (1000, 1001)])
def test_matrix_form_equals_flat_form(eng, nt, ne):
    rng = np.random.RandomState(nt)
    s = np.round(rng.randn(nt * ne), 3).astype(np.float32)
    tl, el = rng.randint(0, 9, nt).astype(np.int32), rng.randint(0, 9, ne).astype(np.int32)
    assert (nt * ne) % TILE != 0
    flat = om.matrix_labels(tl, el)
    rm, sm, lm = eng.verify(s, trial_labels=tl, enroll_labels=el, sorted_out=True)
    rf, sf, lf = eng.verify(s, labels=flat, sorted_out=True)
    assert bytes(rm) == bytes(rf)
    assert torch.equal(sm, sf) and torch.equal(lm, lf)
    _same_result(rm, om.verify(s, flat)[0])


def test_two_calls_are_bit_identical(eng):
    s, lab = _scores('ties', (1 << 20) + 3, seed=5)
    a = eng.verify(s, labels=lab, sorted_out=True)
    b = eng.verify(s, labels=lab, sorted_out=True)
    assert bytes(a[0]) == bytes(b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


@pytest.mark.parametrize('case', ['no_targets', 'no_impostors', 'empty', 'one_target_lowest', 'one_impostor_lowest'])
def test_index_errors(eng, case):
    s = np.array([0.1, 0.2, 0.3, 0.4, 0.5], dtype=np.float32)
    lab = {'no_targets': [0, 0, 0, 0, 0], 'no_impostors': [1, 1, 1, 1, 1], 'empty': [],
           'one_target_lowest': [1, 0, 0, 0, 0], 'one_impostor_lowest': [0, 1, 1, 1, 1]}[case]
    lab = np.array(lab, dtype=np.int32)
    with pytest.raises(IndexError):
        eng.verification_metrics(s[:len(lab)], labels=lab)


def _host_stable_triple(scores, labels):
    from mvector.metric.metrics import compute_dcf, compute_eer
    order = np.argsort(scores, kind='stable')
    lab = labels[order]
    fnr = np.cumsum(lab == 1) / np.float64((lab == 1).sum())
    fpr = 1 - np.cumsum(lab == 0) / np.float64((lab == 0).sum())
    x1 = np.flatnonzero(fnr - fpr >= 0)[0]
    return float(compute_eer(fnr, fpr)), float(compute_dcf(fnr, fpr)), float(scores[order][x1])


def test_evaluate_sized_run_matches_stable_host_mirror(eng):
    rng = np.random.RandomState(7)
    n, D, spk = 4096, 192, 400
    cen = rng.randn(spk, D)
    tl, el = rng.randint(0, spk, n).astype(np.int32), rng.randint(0, spk, n).astype(np.int32)
    trials = (cen[tl] + 1.5 * rng.randn(n, D)).astype(np.float32)
    enroll = (cen[el] + 1.5 * rng.randn(n, D)).astype(np.float32)
    S = eng.cosine_scores(trials, enroll)
    got = eng.verification_metrics(S.reshape(-1), trial_labels=tl, enroll_labels=el)
    want = _host_stable_triple(S.cpu().numpy().reshape(-1), om.matrix_labels(tl, el))
    assert got == want


def test_curves_match_compute_fnr_fpr(eng):
    """curves=True on the reference evaluate's own (tie-free) score list: fnr / fpr / thresholds bit-identical to
    compute_fnr_fpr, and the triple to compute_eer / compute_dcf."""
    from mvector.metric.metrics import compute_dcf, compute_eer, compute_fnr_fpr
    z = np.load(os.path.join(GOLDEN, 'evaluate_small.npz'))
    eer, dcf, thr, fnr, fpr, th = eng.verification_metrics(z['scores'], labels=z['labels'], curves=True)
    fnr_h, fpr_h, th_h = compute_fnr_fpr(z['scores'], z['labels'])
    assert np.array_equal(fnr, fnr_h) and np.array_equal(fpr, fpr_h) and np.array_equal(th, th_h)
    eer_h, thr_h = compute_eer(fnr_h, fpr_h, z['scores'])
    assert (eer, dcf, thr) == (float(eer_h), float(compute_dcf(fnr_h, fpr_h)), float(thr_h))


def _evaluate_on_device(tmp_path, manifest, monkeypatch, save_image_path=None):
    from mvector.trainer import MVectorTrainer
    m = manifest['evaluate_small']
    z = np.load(os.path.join(GOLDEN, 'evaluate_small.npz'))
    lists = {}
    for nm, count in (('enroll', m['n_enroll']), ('trials', m['n_trials'])):
        lines = []
        for i in range(count):
            p = tmp_path / f'{nm}_{i}.wav'
            with wave.open(str(p), 'wb') as w:
                w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000)
                w.writeframes(z[f'{nm}_pcm{i}'].astype('<i2').tobytes())
            lines.append(f'{p}\t{int(z[f"{nm}_label{i}"])}\n')
        lp = tmp_path / f'{nm}_list.txt'
        lp.write_text(''.join(lines))
        lists[nm] = str(lp)
    sd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith('sd/')}
    mdir = tmp_path / 'model'
    mdir.mkdir()
    torch.save({'0.' + k: v for k, v in sd.items()}, str(mdir / 'model.pth'))
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': True, 'target_dB': -20},
                            'eval_conf': dict(m['eval_conf']), 'enroll_list': lists['enroll'],
                            'trials_list': lists['trials']},
           'preprocess_conf': {'feature_method': 'Fbank', 'method_args': dict(m['preprocess']['method_args'])},
           'model_conf': {'model': m['model'], 'model_args': dict(m['model_args'])}}
    monkeypatch.setattr(MVectorTrainer, 'DEVICE_METRICS_MIN', 0)
    import mvector.trainer as mt
    monkeypatch.setattr(mt, 'compute_fnr_fpr', lambda *a, **k: pytest.fail('host metric path taken'))
    eer, min_dcf, thr = MVectorTrainer(cfg, use_gpu=True).evaluate(resume_model=str(mdir), save_image_path=save_image_path)
    assert abs(eer - float(z['eer'])) < 1e-6 and abs(min_dcf - float(z['min_dcf'])) < 1e-6
    assert abs(thr - float(z['threshold'])) < 2e-5


def test_evaluate_on_device_matches_reference_golden(tmp_path, manifest, monkeypatch):
    """MVectorTrainer.evaluate with the device metrics forced on (DEVICE_METRICS_MIN = 0) on the reference's evaluate
    set (tests/golden/evaluate_small.npz): the same EER / minDCF / threshold as the host path reaches."""
    _evaluate_on_device(tmp_path, manifest, monkeypatch)


def test_evaluate_on_device_writes_the_plot(tmp_path, manifest, monkeypatch):
    pytest.importorskip('matplotlib')
    _evaluate_on_device(tmp_path, manifest, monkeypatch, save_image_path=str(tmp_path / 'img'))
    assert (tmp_path / 'img' / 'result.png').stat().st_size > 0
