"""Spectral stage of the diarization clustering on the device (csrc/spectral.cu through vp_spectral_laplacian /
vp_sym_tridiag / vp_sym_tridiag_apply_q) against the fp64 oracle (oracle/spectral.py), numpy.linalg.eigh and the
reference's own outputs."""
import os
import tempfile

import numpy as np
import pytest
import scipy.linalg
import torch

from conftest import GOLDEN, load_golden
from oracle import spectral as osp

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    e = Engine()
    yield e
    e.close()


def _clustered(n, seed, spk=5, dim=48):
    rng = np.random.RandomState(seed)
    cen = rng.randn(spk, dim)
    return (cen[rng.randint(0, spk, n)] + 0.7 * rng.randn(n, dim)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ Laplacian
@pytest.mark.parametrize('n', [1, 4, 5, 6, 7, 272, 273, 300, 2500])
def test_laplacian_matches_oracle(eng, n):
    X = _clustered(n, seed=n)
    _check_laplacian(eng, X)


def test_laplacian_exact_ties_at_the_cut(eng):
    """Rows repeated many times give bit-identical cosines: the cut falls inside runs of equal values, where the
    lower column indices must be the ones dropped."""
    base = _clustered(20, seed=3)
    X = base[np.random.RandomState(4).randint(0, 20, 300)]
    S = eng.cosine_scores(X, X).cpu().numpy()
    nd = osp.n_drop(300)
    srt = np.sort(S, axis=1)
    assert (srt[:, nd - 1] == srt[:, nd]).sum() > 100             # most rows have a tie across the cut
    _check_laplacian(eng, X)


def _check_laplacian(eng, X):
    n = X.shape[0]
    nd = osp.n_drop(n)
    S = eng.cosine_scores(X, X).cpu().numpy()                    # the same kernel vp_spectral_laplacian starts with
    ref = osp.laplacian(osp.prune(S, nd))
    got = eng.spectral_laplacian(X, nd).cpu().numpy()
    assert got.dtype == np.float64 and got.shape == (n, n)
    off = ~np.eye(n, dtype=bool)
    assert np.array_equal((got != 0) & off, (ref != 0) & off)   # the pruning mask, exactly
    assert np.array_equal(got, got.T)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()


def test_laplacian_rejects_bad_arguments(eng):
    from mvector import _lib as L
    X = _clustered(10, seed=1)
    for nd in (-1, 10):
        with pytest.raises(L.VpError) as ei:
            eng.spectral_laplacian(X, nd)
        assert ei.value.code == L.VP_ERR_INVALID
    A = eng.spectral_laplacian(X, 2)
    d, e, tau = eng.sym_tridiag(A)
    with pytest.raises(L.VpError):
        eng.sym_tridiag_apply_q(A, tau, np.zeros((10, 11)))


# ------------------------------------------------------------------------------------------------ eigen stage
def _eig_checks(Lh, lam, Z):
    k = Z.shape[1]
    norm1 = np.abs(Lh).sum(axis=0).max()
    lam_np = np.linalg.eigvalsh(Lh)[:k]
    assert np.abs(lam[:k] - lam_np).max() <= 1e-10 * norm1, np.abs(lam[:k] - lam_np).max() / norm1
    assert np.abs(Lh @ Z - Z * lam[:k]).max() <= 1e-9 * norm1
    assert np.abs(Z.T @ Z - np.eye(k)).max() <= 1e-10


def _device_eig(eng, Ld, k):
    A = Ld.clone()
    d, e, tau = eng.sym_tridiag(A)
    dh, eh = d.cpu().numpy(), e.cpu().numpy()
    lam, Zt = osp.tridiag_eig(dh, eh, k)
    Z = eng.sym_tridiag_apply_q(A, tau, Zt).cpu().numpy()
    return dh, eh, lam, Z


@pytest.mark.parametrize('n', [7, 64, 300, 1000, 2500, 4100])
def test_tridiag_eigenpairs(eng, n):
    X = _clustered(n, seed=100 + n)
    Ld = eng.spectral_laplacian(X, osp.n_drop(n))
    Lh = Ld.cpu().numpy()
    k = min(n, 16)
    d1, e1, lam, Z1 = _device_eig(eng, Ld, k)
    _eig_checks(Lh, lam, Z1)
    d2, e2, _, Z2 = _device_eig(eng, Ld, k)                      # bit-reproducible
    assert np.array_equal(d1, d2) and np.array_equal(e1, e2) and np.array_equal(Z1, Z2)


def test_tridiag_three_components(eng):
    """Three disconnected graphs, interleaved by a permutation: eigenvalue 0 has multiplicity 3, so only the residual
    and orthogonality of the eigenvectors are checked, not the vectors."""
    blocks = [osp.laplacian(osp.prune(osp.cosine(_clustered(m, seed=m)), osp.n_drop(m))) for m in (90, 160, 250)]
    Lh = scipy.linalg.block_diag(*blocks)
    perm = np.random.RandomState(0).permutation(Lh.shape[0])
    Lh = np.ascontiguousarray(Lh[perm][:, perm])
    _, _, lam, Z = _device_eig(eng, torch.from_numpy(Lh).cuda(), 16)
    assert np.abs(lam[:3]).max() <= 1e-10 * np.abs(Lh).sum(axis=0).max()
    _eig_checks(Lh, lam, Z)


def test_spectral_embedding_small_sizes(eng):
    for n in (1, 2, 3):
        X = _clustered(n, seed=n)
        lam, Z = eng.spectral_embedding(X, osp.n_drop(n), n, lambda lam: 1)
        assert lam.shape == (n,) and Z.shape == (n, 1) and abs(np.linalg.norm(Z) - 1) < 1e-12


# ------------------------------------------------------------------------------------------------ end to end
def _device_sd(eng):
    from mvector.infer_utils.speaker_diarization import SpeakerDiarization
    sd = SpeakerDiarization()
    sd.set_spectral(eng.spectral_embedding)
    return sd


def test_device_clustering_reproduces_diarization_golden(eng):
    z = np.load(os.path.join(GOLDEN, 'diarization.npz'))
    sd = _device_sd(eng)
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
def test_device_clustering_reproduces_large_golden(eng, case):
    from mvector.infer_utils.speaker_diarization import SpectralCluster
    z = np.load(os.path.join(GOLDEN, 'spectral_large.npz'))
    X = z[f'{case}/X']
    sd = _device_sd(eng)
    for tag, k in (('auto', None), ('k2', 2), ('k3', 3)):
        sc = SpectralCluster()
        sc.spectral_fn = eng.spectral_embedding
        np.random.seed(0)
        labels = sc(X.copy(), oracle_num=k)
        assert np.array_equal(labels, z[f'{case}/labels_{tag}']), tag
        if tag == 'auto':
            assert labels.max() + 1 == int(z[f'{case}/num_spk'])
        np.random.seed(0)
        sd_labels, centres = sd.clustering(X.copy(), speaker_num=k)
        assert np.array_equal(sd_labels, z[f'{case}/sd_labels_{tag}']), tag
        assert np.allclose(centres, z[f'{case}/centres_{tag}'], atol=1e-6), tag


def test_predictor_diarization_device_equals_host_path(manifest):
    """Ten minutes of four alternating synthetic voices: MVectorPredictor.speaker_diarization with the device spectral
    stage returns exactly what the host path (hook removed) returns, under the same np.random seed."""
    from mvector.predict import MVectorPredictor
    m = manifest['ecapa_small']
    _, sd = load_golden('ecapa_small')
    cfg = {'dataset_conf': {'dataset': {'min_duration': 0.3, 'max_duration': 3, 'sample_rate': 16000,
                                        'use_dB_normalization': False, 'target_dB': -20}},
           'preprocess_conf': {'use_hf_model': False, 'feature_method': m['preprocess']['feature_method'],
                               'method_args': dict(m['preprocess']['method_args'])},
           'model_conf': {'model': m['model'], 'model_args': dict(m['model_args'])}}
    with tempfile.TemporaryDirectory() as td:
        torch.save({'0.' + k: v for k, v in sd.items()}, os.path.join(td, 'model.pth'))
        pred = MVectorPredictor(configs=cfg, model_path=td, use_gpu=True)
    rng = np.random.RandomState(21)
    voices = [(105.0, 0.6), (165.0, 0.35), (240.0, 0.8), (330.0, 0.5)]        # (f0, harmonic decay)

    def voice(f0, decay, n, seed):
        t = np.arange(n) / 16000.0
        x = sum(decay ** h * np.sin(2 * np.pi * f0 * (h + 1) * t) for h in range(10))
        return 0.1 * x / np.abs(x).max() + 0.01 * np.random.RandomState(seed).randn(n)

    parts, total, i = [], 0, 0
    while total < 600 * 16000:
        n = int(rng.uniform(4.0, 12.0) * 16000)
        parts += [voice(*voices[i % 4], n, i), np.zeros(6400)]
        total += n + 6400
        i += 1
    x = np.concatenate(parts).astype(np.float32)
    assert pred.speaker_diarize.spectral_cluster.spectral_fn is not None
    np.random.seed(0)
    dev = pred.speaker_diarization(x, sample_rate=16000)
    pred.speaker_diarize.set_spectral(None)
    np.random.seed(0)
    host = pred.speaker_diarization(x, sample_rate=16000)
    print('segments', len(dev), 'speakers', sorted({o['speaker'] for o in dev}))
    assert len(dev) > 20 and dev == host
