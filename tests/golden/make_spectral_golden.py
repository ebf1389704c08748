"""Generate tests/golden/spectral_large.npz with the UNMODIFIED reference's SpectralCluster
(mvector/infer_utils/speaker_diarization.py:219-310) on seeded synthetic speaker embeddings at sizes where the spectral
stage is not trivial.  Needs the reference checkout (see make_golden.py); run from the repository root:
    python tests/golden/make_spectral_golden.py

Cases: 'six' = 1500 chunks x 64 dims, 6 speakers; 'three' = 600 x 64, 3 speakers.  Speakers take turns in runs of
3..24 chunks; an embedding is its speaker's centre plus isotropic noise, projected on the unit sphere, and a chunk at a
change of speaker mixes the two centres.  The speaker
centres are built in a hierarchy (pairs of close speakers, two of the pairs closer than the third) so that the
Laplacian's smallest eigenvalues are distinct and the k = 2 and k = 3 partitions are well posed as well as the automatic
one.  Stored per case: the inputs, the reference's 16 smallest eigenvalues (float32, as its eigh returns them), the
automatic speaker count and SpectralCluster's labels for auto / k=2 / k=3 under np.random.seed(0), plus
SpeakerDiarization.clustering's relabelled labels and centres; the parameters of each case and its eigengap margin go
to spectral_large.json.  The script refuses ill-posed cases: float64
numpy.linalg.eigh must give the same labels as the reference's float32 path, and the largest eigengap must beat the
runner-up by GAP_MARGIN."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import install_yeaudio_stub  # noqa: E402  (puts the reference first on sys.path)

GAP_MARGIN = 2.0
CASES = {   # name: (n, dims, hierarchy of centre offsets, noise, seed)
    'six': (1500, 64, 6, 0.5, 11),
    'three': (600, 64, 3, 0.5, 12),
}


def make_embeddings(n, dim, spk, noise, seed):
    rng = np.random.RandomState(seed)
    if spk == 6:       # ((0 1) (2 3)) (4 5)
        top = rng.randn(2, dim)
        mid = np.stack([top[0] + 0.6 * rng.randn(dim), top[0] + 0.6 * rng.randn(dim), top[1] + 0.6 * rng.randn(dim)])
        cen = np.stack([mid[i // 2] + 0.45 * rng.randn(dim) for i in range(6)])
    else:              # (0 1) 2
        top = rng.randn(2, dim)
        cen = np.stack([top[0] + 0.55 * rng.randn(dim), top[0] + 0.55 * rng.randn(dim), top[1]])
    cen /= np.linalg.norm(cen, axis=1, keepdims=True)
    # the next speaker follows the same hierarchy: mostly the partner of a pair, rarely the other top-level group
    pair = np.arange(spk) // 2
    top = (pair >= 2).astype(int) if spk == 6 else (pair >= 1).astype(int)
    w = np.where(pair[:, None] == pair[None, :], 8.0, np.where(top[:, None] == top[None, :], 2.0, 0.5))
    np.fill_diagonal(w, 0.0)
    turn = []
    s = 0
    while len(turn) < n:
        turn += [s] * int(rng.randint(3, 25))
        s = int(rng.choice(spk, p=w[s] / w[s].sum()))
    turn = np.array(turn[:n])
    x = cen[turn] + noise / np.sqrt(dim) * rng.randn(n, dim)
    # a chunk that straddles a change of speaker carries some of both voices: these bridge the speakers' graphs
    change = np.flatnonzero(turn[1:] != turn[:-1]) + 1
    mix = rng.uniform(0.3, 0.7, change.size)[:, None]
    x[change] = mix * cen[turn[change]] + (1 - mix) * cen[turn[change - 1]] + noise / np.sqrt(dim) * rng.randn(change.size, dim)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return x.astype(np.float32), turn


def main():
    install_yeaudio_stub()
    import scipy.linalg
    from mvector.infer_utils.speaker_diarization import SpectralCluster, SpeakerDiarization
    out = {}
    manifest_entry = {}
    for name, (n, dim, spk, noise, seed) in CASES.items():
        X, turn = make_embeddings(n, dim, spk, noise, seed)
        sc = SpectralCluster()
        A = sc.p_pruning(sc.get_sim_mat(X))
        Lf = sc.get_laplacian(0.5 * (A + A.T))
        assert Lf.dtype == np.float32
        lam = scipy.linalg.eigh(Lf, eigvals_only=True)[:16]
        # float64 restatement for the well-posedness checks
        L64 = Lf.astype(np.float64)
        lam64, vec64 = np.linalg.eigh(L64)
        gaps = np.diff(lam64[:16])
        order = np.sort(gaps)[::-1]
        assert order[0] > GAP_MARGIN * order[1], (name, gaps)
        # connected graph, and every k used below separated from the next eigenvalue: the spectral embedding is
        # determined up to signs, not just up to a rotation inside a repeated eigenvalue
        for k in (2, 3, spk):
            assert lam64[k] - lam64[k - 1] > 0.2 * lam64[k], (name, k, lam64[:8])
        out[f'{name}/X'] = X
        out[f'{name}/turn'] = turn.astype(np.int16)
        out[f'{name}/lambdas'] = lam.astype(np.float32)
        for tag, k in (('auto', None), ('k2', 2), ('k3', 3)):
            np.random.seed(0)
            labels = SpectralCluster()(X.copy(), oracle_num=k)
            kk = int(labels.max()) + 1
            np.random.seed(0)
            ref64 = SpectralCluster.cluster_embs(vec64[:, :kk].astype(np.float32), kk)
            assert np.array_equal(labels, ref64), (name, tag)
            np.random.seed(0)
            sd_labels, centres = SpeakerDiarization().clustering(X.copy(), speaker_num=k)
            out[f'{name}/labels_{tag}'] = np.asarray(labels, dtype=np.int64)
            out[f'{name}/sd_labels_{tag}'] = np.asarray(sd_labels, dtype=np.int64)
            out[f'{name}/centres_{tag}'] = np.asarray(centres, dtype=np.float32)
            if tag == 'auto':
                out[f'{name}/num_spk'] = np.int32(kk)
                assert kk == spk, (name, kk)
            print(name, tag, kk, np.bincount(labels), 'sd speakers', sd_labels.max() + 1)
        manifest_entry[name] = dict(n=n, dim=dim, speakers=spk, noise=noise, seed=seed,
                                    largest_gap_over_runner_up=float(order[0] / order[1]))
    path = os.path.join(HERE, 'spectral_large.npz')
    np.savez_compressed(path, **out)
    print('spectral_large.npz', os.path.getsize(path) // 1024, 'KiB')
    # the fixture's description sits next to it (manifest.json describes the fixtures of make_golden.py)
    meta = dict(note='reference SpectralCluster / SpeakerDiarization.clustering on seeded clustered unit-sphere '
                     'embeddings (tests/golden/make_spectral_golden.py; np.random.seed(0) before every k_means)',
                cases=manifest_entry)
    with open(os.path.join(HERE, 'spectral_large.json'), 'w') as f:
        json.dump(meta, f, indent=1, sort_keys=True)
        f.write('\n')

if __name__ == '__main__':
    main()
