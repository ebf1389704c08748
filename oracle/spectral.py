"""numpy fp64 restatement of the device spectral stage (voiceprintrecognition-pytorch_b200/csrc/spectral.cu), stage by
stage, for the tests: the p_pruning count, the stable-tie pruning, the Laplacian, the dsytd2-convention Householder
reduction (d, e, tau, reflectors in the strictly lower part) and the back-transformation Z <- Q Z.

Reference: mvector/infer_utils/speaker_diarization.py:235-310 (SpectralCluster)."""
import numpy as np
import scipy.linalg


def n_drop(n, pval=0.022):
    """Entries p_pruning (:260-274) zeroes per row of an n x n affinity: ``argsort(row)[0:int((1 - pval) * n)]`` with
    pval raised to 6/n for small n, as Python evaluates it -- a negative bound slices from the end."""
    p = 6.0 / n if n * pval < 6 else pval
    return len(range(n)[:int((1 - p) * n)])


def cosine(X):
    """float32 cosine matrix as sklearn's cosine_similarity forms it (normalise, then one matmul)."""
    X = np.asarray(X, dtype=np.float32)
    nrm = np.linalg.norm(X, axis=1, keepdims=True)
    Xn = X / np.where(nrm == 0, 1, nrm)
    return Xn @ Xn.T


def prune(A, nd):
    """Zero the nd smallest entries of every row; ties go by column index (stable argsort).  Returns a copy."""
    P = np.array(A, copy=True)
    if nd > 0:
        drop = np.argsort(P, axis=1, kind='stable')[:, :nd]
        np.put_along_axis(P, drop, 0, axis=1)
    return P


def laplacian(P):
    """S = 0.5 (P + P') in fp64 with a zero diagonal, L = diag(sum_j |S_ij|) - S (get_laplacian, :277-283)."""
    P = np.asarray(P, dtype=np.float64)
    S = 0.5 * (P + P.T)
    np.fill_diagonal(S, 0.0)
    return np.diag(np.abs(S).sum(axis=1)) - S


def tridiag(L):
    """LAPACK dsytd2 (UPLO='L') in the device's arithmetic: -> (A with d/e on the diagonals and the reflectors below,
    d [n], e [n-1], tau [n-1]).  The rank-2 update is the exactly symmetric v w' + w v'."""
    A = np.array(L, dtype=np.float64, copy=True)
    n = A.shape[0]
    d = np.zeros(n)
    e = np.zeros(max(n - 1, 0))
    tau = np.zeros(max(n - 1, 0))
    for k in range(n - 1):
        d[k] = A[k, k]
        if k == n - 2:
            e[k] = A[k + 1, k]
            break
        alpha, x = A[k + 1, k], A[k + 2:, k]
        sig = float(np.dot(x, x))
        if sig == 0.0:
            beta, t, scal = alpha, 0.0, 0.0
        else:
            beta = -np.copysign(np.sqrt(alpha * alpha + sig), alpha)
            t = (beta - alpha) / beta
            scal = 1.0 / (alpha - beta)
        v = np.concatenate([[1.0], x * scal])
        A[k + 2:, k] = v[1:]
        A[k + 1, k] = beta
        e[k], tau[k] = beta, t
        T = A[k + 1:, k + 1:]
        xw = t * (T @ v)
        w = xw + (-0.5 * t * np.dot(xw, v)) * v
        s = np.outer(v, w)
        s += s.T.copy()
        T -= s
    d[n - 1] = A[n - 1, n - 1]
    return A, d, e, tau


def apply_q(A, tau, Z):
    """Z [n, k] <- H_0 H_1 ... H_{n-3} Z (dorm2r order: the last reflector first)."""
    Z = np.array(Z, dtype=np.float64, copy=True)
    n = A.shape[0]
    for k in range(n - 3, -1, -1):
        v = np.concatenate([[1.0], A[k + 2:, k]])
        w = v @ Z[k + 1:]
        Z[k + 1:] += np.outer(v, -tau[k] * w)
    return Z


def tridiag_eig(d, e, n_eig, vectors=True):
    """The n_eig smallest eigenvalues (and eigenvectors) of tridiag(d, e) (LAPACK stebz / stein)."""
    if d.shape[0] == 1:
        return (d.copy(), np.ones((1, 1))) if vectors else d.copy()
    return scipy.linalg.eigh_tridiagonal(d, e, eigvals_only=not vectors, select='i', select_range=(0, n_eig - 1))


def spectral_embedding(X, nd, n_eig, k_fn):
    """The whole device stage on the CPU, with the interface of SpectralCluster's spectral hook."""
    L = laplacian(prune(cosine(X), nd))
    A, d, e, tau = tridiag(L)
    lam = tridiag_eig(d, e, n_eig, vectors=False)
    k = k_fn(lam)
    _, Zt = tridiag_eig(d, e, k)
    return lam, apply_q(A, tau, Zt)
