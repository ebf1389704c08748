"""CPU checks of the device verification metrics' contract: the numpy restatement of csrc/verify.cu (oracle/metrics.py)
against the host metric functions (mvector/metric/metrics.py) and the reference's golden, the key order, the IndexError
cases, evaluate's routing between the host and device paths, and the ctypes mirror of vp_verify_result."""
import ctypes
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN, ROOT
from oracle import metrics as om


def _host_stable(scores, labels, p_target=0.01, c_miss=1, c_fa=1):
    """compute_fnr_fpr with a stable argsort, then the host compute_eer / compute_dcf."""
    from mvector.metric.metrics import compute_dcf, compute_eer
    order = np.argsort(scores, kind='stable')
    lab = labels[order]
    tgt = np.where(lab == 1, 1.0, 0.0)
    imp = np.where(lab == 0, 1.0, 0.0)
    fnr = np.cumsum(tgt) / np.sum(tgt)
    fpr = 1 - np.cumsum(imp) / np.sum(imp)
    eer = compute_eer(fnr, fpr)
    thr = np.sort(scores)[np.flatnonzero(fnr - fpr >= 0)[0]]
    return fnr, fpr, float(eer), float(compute_dcf(fnr, fpr, p_target, c_miss, c_fa)), float(thr)


def _reference_dcf(fnr, fpr, p_target, c_miss, c_fa):
    """The reference's compute_dcf expression (metrics.py:36-39) literally: c_miss * fnr * p_target + ..."""
    c_det = min(c_miss * fnr * p_target + c_fa * fpr * (1 - p_target))
    return c_det / min(c_miss * p_target, c_fa * (1 - p_target))


def _oracle(scores, labels, **kw):
    from mvector.metric.verification import curves_from_sorted, metrics_from_result
    res, keys, codes = om.verify(scores, labels, **kw)
    fnr, fpr, _ = curves_from_sorted(om.key_scores(keys), codes)
    return res, fnr, fpr, metrics_from_result(res, **kw)


@pytest.mark.parametrize('n,seed', [(3, 0), (57, 1), (4096, 2), (20001, 3)])
def test_oracle_bit_identical_to_host_on_tie_free_lists(n, seed):
    from mvector.metric.metrics import compute_dcf, compute_eer, compute_fnr_fpr
    rng = np.random.RandomState(seed)
    scores = rng.permutation(np.linspace(-1, 1, n, dtype=np.float32))        # distinct values
    labels = (rng.rand(n) < 0.3).astype(np.int32)
    labels[np.argmin(scores)], labels[np.argmax(scores)] = 0, 1
    assert len(np.unique(scores)) == n
    fnr_h, fpr_h, th_h = compute_fnr_fpr(scores, labels)
    res, fnr, fpr, (eer, dcf, thr) = _oracle(scores, labels)
    assert np.array_equal(fnr, fnr_h) and np.array_equal(fpr, fpr_h)
    eer_h, thr_h = compute_eer(fnr_h, fpr_h, scores)
    assert eer == float(eer_h) and thr == float(thr_h)
    assert dcf == float(compute_dcf(fnr_h, fpr_h))
    for kw in (dict(p_target=0.05, c_miss=10, c_fa=1), dict(p_target=0.3, c_miss=1, c_fa=3.5)):
        res, fnr, fpr, (eer, dcf, thr) = _oracle(scores, labels, **kw)
        assert dcf == float(_reference_dcf(fnr_h, fpr_h, **kw))
        assert abs(dcf - float(compute_dcf(fnr_h, fpr_h, **kw))) <= 1e-15 * abs(dcf)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_oracle_with_ties_equals_stable_order_host(seed):
    rng = np.random.RandomState(seed)
    n = 9000
    scores = np.round(rng.randn(n) * 0.3, 2).astype(np.float32)              # ~200 distinct values: heavy ties
    labels = (rng.rand(n) < 0.2).astype(np.int32)
    fnr_h, fpr_h, eer_h, dcf_h, thr_h = _host_stable(scores, labels)
    res, fnr, fpr, (eer, dcf, thr) = _oracle(scores, labels)
    assert np.array_equal(fnr, fnr_h) and np.array_equal(fpr, fpr_h)
    assert (eer, dcf, thr) == (eer_h, dcf_h, thr_h)
    kw = dict(p_target=0.05, c_miss=10, c_fa=1)
    assert _oracle(scores, labels, **kw)[3][1] == float(_reference_dcf(fnr_h, fpr_h, **kw))


def test_oracle_against_reference_golden():
    """tests/golden/metrics.npz (scores rounded to 3 decimals, made by the reference's own functions): threshold and
    minDCF equal; the EER may move within the tie group at the crossing, at most (group size) / min(T, I)."""
    z = np.load(os.path.join(GOLDEN, 'metrics.npz'))
    scores, labels = z['scores'], z['labels']
    res, fnr, fpr, (eer, dcf, thr) = _oracle(scores, labels)
    assert thr == float(z['threshold'])
    assert abs(dcf - float(z['min_dcf'])) < 1e-12
    # at (0.05, 10, 1) the cost minimum falls inside a tie group: it may move by the cost of reordering that group
    res05, _, _, (_, dcf05, _) = _oracle(scores, labels, p_target=0.05, c_miss=10, c_fa=1)
    g = int((scores == om.key_scores(om.stable_sort(scores, labels)[0][res05.argmin:res05.argmin + 1])[0]).sum())
    step = (10 * 0.05 / res05.n_target + 1 * 0.95 / res05.n_impostor) / min(10 * 0.05, 0.95)
    assert 0 < abs(dcf05 - float(z['min_dcf_05'])) <= g * step
    group = int((scores == np.float32(thr)).sum())
    bound = group / min(res.n_target, res.n_impostor)
    assert abs(eer - float(z['eer'])) <= bound, (eer, float(z['eer']), bound)


def test_key_order_matches_numpy_sort():
    sub = np.float32(1e-45)
    x = np.array([np.nan, 1.0, -0.0, 0.0, -np.inf, np.inf, sub, -sub, -1.0, np.float32(3e38), -np.float32(3e38),
                  np.float32(1.2e-38), -np.float32(1.2e-38), -np.nan, 0.5, -0.5, 0.0, -0.0, np.nan], dtype=np.float32)
    x = np.concatenate([x, np.random.RandomState(0).randn(200).astype(np.float32)])
    keys = om.score_keys(x)
    order = np.argsort(keys, kind='stable')
    got = x[order]
    want = np.sort(x, kind='stable')
    assert np.array_equal(got, want, equal_nan=True)                  # -0 == +0 compare equal
    assert np.array_equal(order, np.argsort(x, kind='stable'))        # including the order within the ties
    assert keys[np.isnan(x)].min() > keys[x == np.inf].max()
    assert len(set(keys[x == 0].tolist())) == 1
    dec = om.key_scores(keys)
    fin = ~np.isnan(x)
    assert np.array_equal(dec[fin], np.where(x[fin] == 0, np.float32(0), x[fin]))


@pytest.mark.parametrize('case', ['no_targets', 'no_impostors', 'empty', 'one_target_lowest', 'one_impostor_lowest'])
def test_index_errors_match_host(case):
    from mvector.metric.metrics import compute_eer, compute_fnr_fpr
    from mvector.metric.verification import metrics_from_result
    s = np.array([0.1, 0.2, 0.3, 0.4, 0.5], dtype=np.float32)
    lab = {'no_targets': [0, 0, 0, 0, 0], 'no_impostors': [1, 1, 1, 1, 1], 'empty': [],
           'one_target_lowest': [1, 0, 0, 0, 0], 'one_impostor_lowest': [0, 1, 1, 1, 1]}[case]
    lab = np.array(lab, dtype=np.int32)
    s = s[:len(lab)]
    with pytest.raises(IndexError), np.errstate(all='ignore'):
        compute_eer(*compute_fnr_fpr(s, lab)[:2])
    res = om.verify(s, lab)[0]
    with pytest.raises(IndexError):
        metrics_from_result(res)


# ------------------------------------------------------------------------------------------------ evaluate routing
class _StubEngine:
    def __init__(self):
        self.calls = []

    def cosine_scores(self, a, b):
        import torch
        return torch.from_numpy(_cos(a, b))

    def verification_metrics(self, scores_dev, labels=None, trial_labels=None, enroll_labels=None, p_target=0.01,
                             c_miss=1, c_fa=1, curves=False):
        from mvector.metric.verification import metrics_from_result
        self.calls.append(dict(n=scores_dev.numel(), trial_labels=np.asarray(trial_labels),
                               enroll_labels=np.asarray(enroll_labels), curves=curves))
        lab = om.matrix_labels(trial_labels, enroll_labels)
        return metrics_from_result(om.verify(scores_dev.numpy(), lab, p_target, c_miss, c_fa)[0], p_target, c_miss, c_fa)


def _cos(a, b):
    an = a / np.linalg.norm(a, axis=1, keepdims=True)
    bn = b / np.linalg.norm(b, axis=1, keepdims=True)
    return (an @ bn.T).astype(np.float32)


def _trainer(n_trials, n_enroll, seed=0):
    import mvector.trainer as mt
    from mvector.utils.utils import dict_to_object
    rng = np.random.RandomState(seed)
    data = {'enroll': (rng.randn(n_enroll, 16).astype(np.float32), rng.randint(0, 7, n_enroll).astype(np.int32)),
            'trials': (rng.randn(n_trials, 16).astype(np.float32), rng.randint(0, 7, n_trials).astype(np.int32))}
    tr = object.__new__(mt.MVectorTrainer)
    tr.configs = dict_to_object({'dataset_conf': {'enroll_list': 'enroll', 'trials_list': 'trials'}})
    tr.stop_eval = False
    tr.model = type('M', (), {'eval': lambda self: self})()
    tr._engine = _StubEngine()
    tr._embed_list = lambda name: data[name]
    tr._cosine_scores = lambda t, e: _cos(t, e)
    return tr, data


def test_evaluate_routes_small_matrices_to_the_host_path():
    tr, _ = _trainer(30, 40)
    assert tr.DEVICE_METRICS_MIN > 30 * 40
    tr.evaluate()
    assert tr._engine.calls == []


def test_evaluate_routes_large_matrices_to_the_device_with_trial_major_labels():
    tr, data = _trainer(31, 43, seed=1)
    host = tr.evaluate()
    tr.DEVICE_METRICS_MIN = 31 * 43
    dev = tr.evaluate()
    (call,) = tr._engine.calls
    assert call['n'] == 31 * 43 and not call['curves']
    assert np.array_equal(call['trial_labels'], data['trials'][1])
    assert np.array_equal(call['enroll_labels'], data['enroll'][1])
    assert len(np.unique(_cos(data['trials'][0], data['enroll'][0]))) == 31 * 43     # tie-free scores
    assert dev == host


# ------------------------------------------------------------------------------------------------ ctypes mirror
def _header_struct_fields(name):
    src = open(os.path.join(ROOT, 'include', 'vpb200.h')).read()
    body = re.search(r'typedef struct %s \{(.*?)\} %s;' % (name, name), src, re.S).group(1)
    body = re.sub(r'/\*.*?\*/', '', body, flags=re.S)
    fields = []
    for decl in body.split(';'):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(ctype, n.strip()) for n in names.split(',')]
    return fields


def test_verify_result_mirror_follows_the_header():
    from mvector import _lib
    ctype_of = {'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64, 'float': ctypes.c_float, 'double': ctypes.c_double}
    want = _header_struct_fields('vp_verify_result')
    got = list(_lib.VerifyResult._fields_)
    assert [n for _, n in want] == [n for n, _ in got]
    assert [ctype_of[t] for t, _ in want] == [t for _, t in got]
    assert ctypes.sizeof(_lib.VerifyResult) == 88
