"""EER, minDCF and the EER threshold of a verification score list on the GPU (csrc/verify.cu through vp_verify_metrics).

Same definitions as compute_fnr_fpr / compute_eer / compute_dcf (metric/metrics.py), which stay the host path.  The device
sorts the scores with a stable radix sort and reduces the miss / false-alarm curves to a handful of integers and one
cost (vp_verify_result); the scalar EER and minDCF are then formed here, with compute_eer's and compute_dcf's own float64
expressions, so they are bit-identical to the host functions on the same sorted label sequence.  Equal scores keep their
index order (``np.argsort(kind='stable')``); the host path's default quicksort leaves that order open, which can move
the EER within a tie group that straddles the crossing.

    from mvector.metric.verification import verification_metrics
    eer, min_dcf, threshold = verification_metrics(scores, labels)          # numpy / torch scores, 0/1 labels
"""
import numpy as np


def metrics_from_result(res, p_target=0.01, c_miss=1, c_fa=1):
    """(eer, min_dcf, threshold) from a vp_verify_result (any object with its fields).  Raises IndexError where
    compute_eer does: no target, no impostor, no score, or no sorted index with fnr - fpr < 0."""
    n_t, n_i = int(res.n_target), int(res.n_impostor)
    if n_t == 0 or n_i == 0 or res.x1 < 0 or res.x2 < 0:
        why = ('no scores' if n_t + n_i == 0 else 'no target pair' if n_t == 0 else 'no impostor pair' if n_i == 0
               else 'no threshold with fnr < fpr')
        raise IndexError(f'EER undefined: {why} (targets {n_t}, impostors {n_i})')
    T, I = np.float64(n_t), np.float64(n_i)
    fnr1, fpr1 = np.float64(res.target_x1) / T, 1 - np.float64(res.impostor_x1) / I
    fnr2, fpr2 = np.float64(res.target_x2) / T, 1 - np.float64(res.impostor_x2) / I
    a = (fnr1 - fpr1) / (fpr2 - fpr1 - (fnr2 - fnr1))          # compute_eer (metrics.py:23-33), x1 = hi, x2 = lo
    eer = fnr1 + a * (fnr2 - fnr1)
    c_def = min(c_miss * p_target, c_fa * (1 - p_target))      # compute_dcf (metrics.py:36-39)
    return float(eer), float(np.float64(res.min_cost) / c_def), float(res.threshold)


def curves_from_sorted(sorted_scores, sorted_labels):
    """(fnr, fpr, thresholds) as compute_fnr_fpr forms them, from the sorted scores and label codes (1 target, 0
    impostor)."""
    lab = np.asarray(sorted_labels)
    tgt = (lab == 1).astype(np.float64)
    imp = (lab == 0).astype(np.float64)
    fnr = np.cumsum(tgt) / np.sum(tgt)
    fpr = 1 - np.cumsum(imp) / np.sum(imp)
    return fnr, fpr, np.asarray(sorted_scores)


def verification_metrics(scores, labels, p_target=0.01, c_miss=1, c_fa=1, curves=False, engine=None):
    """compute_fnr_fpr + compute_eer + compute_dcf of a flat score list on the GPU -> (eer, min_dcf, threshold), plus
    (fnr, fpr, thresholds) with ``curves=True``.  ``scores``: numpy or torch (a CUDA tensor stays on the device);
    ``labels``: 1 target, 0 impostor.  ``engine``: an mvector.engine.Engine (one is created when None)."""
    if engine is None:
        from ..engine import Engine
        engine = Engine()
    return engine.verification_metrics(scores, labels=labels, p_target=p_target, c_miss=c_miss, c_fa=c_fa, curves=curves)
