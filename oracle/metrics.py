"""numpy restatement of the device verification metrics (voiceprintrecognition-pytorch_b200/csrc/verify.cu) for the
tests: the order-preserving score key (with -0 and NaN folding), the stable sort, the integer prefix counts, x1 / x2 /
the minimum cost and its first index, the cost in numpy's operation order, and the vp_verify_result fields.

Reference: mvector/metric/metrics.py:5-39 (compute_fnr_fpr, compute_eer, compute_dcf)."""
from types import SimpleNamespace

import numpy as np


def score_keys(scores):
    """uint32 keys that order like numpy orders the float32 scores: -0 -> key of +0, every NaN -> 0xffffffff."""
    f = np.asarray(scores, dtype=np.float32).copy()
    f[f == 0] = 0.0
    u = f.view(np.uint32)
    k = np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)
    k[np.isnan(f)] = np.uint32(0xffffffff)
    return k


def key_scores(keys):
    """float32 scores the keys decode to (inverse of score_keys up to the folding)."""
    k = np.asarray(keys, dtype=np.uint32)
    u = np.where(k & np.uint32(0x80000000), k & np.uint32(0x7fffffff), ~k).astype(np.uint32)
    return u.view(np.float32)


def label_codes(labels):
    """Payload the device sorts with the keys: 1 target (label 1), 0 impostor (label 0), 2 neither."""
    lab = np.asarray(labels)
    return np.where(lab == 1, 1, np.where(lab == 0, 0, 2)).astype(np.uint8)


def matrix_labels(trial_labels, enroll_labels):
    """evaluate's trial-major label list: score i = trial i // n_enroll against enrolment i % n_enroll."""
    return (np.asarray(trial_labels)[:, None] == np.asarray(enroll_labels)[None, :]).astype(np.int32).reshape(-1)


def stable_sort(scores, labels):
    """(sorted keys, sorted label codes) of the stable LSD radix sort: np.argsort(kind='stable') of the keys."""
    keys = score_keys(scores)
    order = np.argsort(keys, kind='stable')
    return keys[order], label_codes(labels)[order]


def verify(scores, labels, p_target=0.01, c_miss=1, c_fa=1):
    """vp_verify_result of vp_verify_metrics on a flat score list (plus the sorted keys and label codes)."""
    keys, codes = stable_sort(scores, labels)
    n = len(keys)
    tc = np.cumsum(codes == 1, dtype=np.int64)                # T_i, I_i: inclusive integer prefix counts
    ic = np.cumsum(codes == 0, dtype=np.int64)
    T = int(tc[-1]) if n else 0
    I = int(ic[-1]) if n else 0
    with np.errstate(divide='ignore', invalid='ignore'):
        fnr = tc.astype(np.float64) / np.float64(T)
        fpr = 1.0 - ic.astype(np.float64) / np.float64(I)
        gap = fnr - fpr
        cost = (np.float64(c_miss) * fnr) * np.float64(p_target) + (np.float64(c_fa) * fpr) * (1.0 - float(p_target))
    hi = np.flatnonzero(gap >= 0)
    lo = np.flatnonzero(gap < 0)
    x1 = int(hi[0]) if len(hi) else -1
    x2 = int(lo[-1]) if len(lo) else -1
    finite = ~np.isnan(cost)
    argmin = int(np.flatnonzero(finite)[np.argmin(cost[finite])]) if finite.any() else -1
    res = SimpleNamespace(
        n_target=T, n_impostor=I, x1=x1, x2=x2,
        target_x1=int(tc[x1]) if x1 >= 0 else 0, impostor_x1=int(ic[x1]) if x1 >= 0 else 0,
        target_x2=int(tc[x2]) if x2 >= 0 else 0, impostor_x2=int(ic[x2]) if x2 >= 0 else 0,
        min_cost=float(cost[argmin]) if argmin >= 0 else float('inf'), argmin=argmin,
        threshold=float(key_scores(keys[x1:x1 + 1])[0]) if x1 >= 0 else float('nan'))
    return res, keys, codes
