"""CPU checks of the spectral stage of the diarization clustering: the p_pruning count, the fp64 oracle of the device
stages (oracle/spectral.py) against numpy.linalg.eigh, and SpectralCluster's spectral hook fed by that oracle against
the reference's own outputs (tests/golden/diarization.npz, spectral_large.npz)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import spectral as osp


def _reference_zeroed(n, pval=0.022):
    """Zeros per row after the reference's p_pruning (:260-274), evaluated literally on a matrix without zeros."""
    A = np.random.RandomState(n).rand(n, n).astype(np.float32) + 1.0
    pv = 6. / A.shape[0] if A.shape[0] * pval < 6 else pval
    n_elems = int((1 - pv) * A.shape[0])
    for i in range(A.shape[0]):
        low_indexes = np.argsort(A[i, :])
        low_indexes = low_indexes[0:n_elems]
        A[i, low_indexes] = 0
    counts = (A == 0).sum(axis=1)
    assert (counts == counts[0]).all()
    return int(counts[0])


def test_n_drop_matches_reference_pruning():
    from mvector.infer_utils.speaker_diarization import SpectralCluster
    sc = SpectralCluster()
    assert (osp.n_drop(4), osp.n_drop(5), osp.n_drop(7)) == (2, 0, 1)
    for n in range(1, 601):
        want = _reference_zeroed(n)
        assert osp.n_drop(n) == want, n
        assert sc.n_drop(n) == want, n


def _clustered_laplacian(n, spk, seed, dim=32):
    rng = np.random.RandomState(seed)
    cen = rng.randn(spk, dim)
    X = (cen[rng.randint(0, spk, n)] + 0.6 * rng.randn(n, dim)).astype(np.float32)
    return osp.laplacian(osp.prune(osp.cosine(X), osp.n_drop(n)))


def test_prune_ties_go_by_column_index():
    A = np.array([[1.0, 0.5, 0.5, 0.5, 0.2, 0.5]], dtype=np.float32)
    P = osp.prune(A, 3)                                # drops 0.2, then the two lowest-index 0.5s
    assert P.tolist() == [[1.0, 0.0, 0.0, 0.5, 0.0, 0.5]]


@pytest.mark.parametrize('n', [4, 7, 64, 500])
def test_oracle_tridiag_reproduces_eigh(n):
    L = _clustered_laplacian(n, 3, seed=n)
    assert np.array_equal(L, L.T)
    A, d, e, tau = osp.tridiag(L)
    k = min(n, 16)
    lam, Zt = osp.tridiag_eig(d, e, k)
    Z = osp.apply_q(A, tau, Zt)
    lam_np, vec_np = np.linalg.eigh(L)
    norm1 = np.abs(L).sum(axis=0).max()
    assert np.abs(lam - lam_np[:k]).max() <= 1e-10 * norm1
    assert np.abs(L @ Z - Z * lam).max() <= 1e-9 * norm1
    assert np.abs(Z.T @ Z - np.eye(k)).max() <= 1e-10
    # invariant subspaces: the span of every group of eigenvalues separated from the rest agrees with eigh's
    edges = [0] + [i + 1 for i in range(k - 1) if lam_np[i + 1] - lam_np[i] > 1e-6 * norm1] + [k]
    if k < n and lam_np[k] - lam_np[k - 1] <= 1e-6 * norm1:
        edges = edges[:-1]
    for a, b in zip(edges[:-1], edges[1:]):
        P_ours = Z[:, a:b] @ Z[:, a:b].T
        P_ref = vec_np[:, a:b] @ vec_np[:, a:b].T
        assert np.abs(P_ours - P_ref).max() < 1e-7, (a, b)


_REDUCED = {}


def _oracle_spectral(X, nd, n_eig, k_fn):
    """osp.spectral_embedding, with the O(n^3) reduction of each input done once per session."""
    key = (X.tobytes(), nd)
    if key not in _REDUCED:
        _REDUCED[key] = osp.tridiag(osp.laplacian(osp.prune(osp.cosine(X), nd)))
    A, d, e, tau = _REDUCED[key]
    lam = osp.tridiag_eig(d, e, n_eig, vectors=False)
    _, Zt = osp.tridiag_eig(d, e, k_fn(lam))
    return lam, osp.apply_q(A, tau, Zt)


def _oracle_cluster():
    from mvector.infer_utils.speaker_diarization import SpectralCluster, SpeakerDiarization
    sd = SpeakerDiarization()
    sd.set_spectral(_oracle_spectral)
    assert isinstance(sd.spectral_cluster, SpectralCluster) and sd.spectral_cluster.spectral_fn is not None
    return sd


def test_spectral_hook_reproduces_diarization_golden():
    z = np.load(os.path.join(GOLDEN, 'diarization.npz'))
    sd = _oracle_cluster()
    vad = [[float(z[f'vad{i}_t'][0]), float(z[f'vad{i}_t'][1]), z[f'vad{i}_x']] for i in range(int(z['n_vad']))]
    chunks = sd._chunk(vad)
    for tag, k in (('auto', None), ('k2', 2), ('k3', 3)):
        np.random.seed(0)
        labels, centres = sd.clustering(z['emb'].copy(), speaker_num=k)
        assert np.array_equal(labels, z[f'labels_{tag}']), tag
        assert np.allclose(centres, z[f'centres_{tag}'], atol=1e-6)
        out = sd.postprocess([list(c) for c in chunks], labels)
        got = np.array([[o['speaker'], o['start'], o['end']] for o in out], dtype=np.float64)
        assert np.array_equal(got, z[f'out_{tag}']), tag


@pytest.mark.parametrize('case', ['six', 'three'])
def test_spectral_hook_reproduces_large_golden(case):
    from mvector.infer_utils.speaker_diarization import SpectralCluster
    z = np.load(os.path.join(GOLDEN, 'spectral_large.npz'))
    X = z[f'{case}/X']
    n = X.shape[0]
    # eigenvalues of the fp64 oracle against the reference's float32 eigh
    L = osp.laplacian(osp.prune(osp.cosine(X), osp.n_drop(n)))
    lam, _ = _oracle_spectral(X, osp.n_drop(n), 16, lambda lam: 1)
    assert np.abs(lam - z[f'{case}/lambdas']).max() < 1e-4 * np.abs(L).sum(axis=0).max()
    sd = _oracle_cluster()
    for tag, k in (('auto', None), ('k2', 2), ('k3', 3)):
        sc = SpectralCluster()
        sc.spectral_fn = _oracle_spectral
        np.random.seed(0)
        labels = sc(X.copy(), oracle_num=k)
        assert np.array_equal(labels, z[f'{case}/labels_{tag}']), tag
        if tag == 'auto':
            assert labels.max() + 1 == int(z[f'{case}/num_spk'])
        np.random.seed(0)
        sd_labels, centres = sd.clustering(X.copy(), speaker_num=k)
        assert np.array_equal(sd_labels, z[f'{case}/sd_labels_{tag}']), tag
        assert np.allclose(centres, z[f"{case}/centres_{tag}"], atol=1e-6), tag
