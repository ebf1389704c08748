"""Op-level tests of the cosine score kernel (csrc/pool.cu cosine_scores_kernel through vp_cosine_scores /
Engine.cosine_scores) on the cases of tests/score_cases.py: every element within its a-priori bound of the fp64 oracle,
zero-norm rows scored 0, scores independent of the call shape and of the run, and the two device callers that start from
the kernel -- the diarization Laplacian and evaluate's metrics -- on embeddings with a zero row."""
import numpy as np
import pytest
import torch

import score_cases as sc
from oracle import metrics as om
from oracle import spectral as osp
from test_gpu_metrics import _host_stable_triple
from test_gpu_spectral import _check_laplacian, _clustered

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    e = Engine()
    yield e
    e.close()


def _scores(eng, a, b):
    return eng.cosine_scores(a, b).cpu().numpy()


@pytest.mark.parametrize('case', sc.CASES, ids=lambda c: c['name'])
def test_case_within_bound(eng, case):
    a, b = sc.make(case)
    worst = sc.check(_scores(eng, a, b), a, b)
    print(f"{case['name']}: err / beta {worst:.3f}")


@pytest.mark.parametrize('case', [c for c in sc.CASES if any(sc.zero_rows(c))], ids=lambda c: c['name'])
def test_zero_rows_score_zero(eng, case):
    """A zero-norm row scores +0 against every row, itself included, as sklearn's cosine_similarity scores it."""
    a, b = sc.make(case)
    got = _scores(eng, a, b)
    za, zb = (list(z) for z in sc.zero_rows(case))
    assert not np.isnan(got).any()
    for block in (got[za], got[:, zb]):
        assert np.array_equal(block.view(np.uint32), np.zeros_like(block, dtype=np.uint32))


def test_nan_stays_in_its_row_and_column(eng):
    case = sc.CASE_BY_NAME['nan_rows']
    a, b = sc.make(case)
    got = _scores(eng, a, b)
    want = np.zeros(got.shape, bool)
    want[list(case['nan_a']), :] = True
    want[:, list(case['nan_b'])] = True
    assert np.array_equal(np.isnan(got), want)


@pytest.mark.parametrize('name', ['shape_257x257', 'range_D192', 'zero_both', 'k_D129'])
def test_score_does_not_depend_on_the_call_shape(eng, name):
    """A pair scores bit-identically in the full call, in a 1 x 1 call and in calls whose other rows and columns put it
    at another place in its tile (retrieval scores one query or a batch; the diarization ties rely on equal rows giving
    equal cosines)."""
    a, b = sc.make(sc.CASE_BY_NAME[name])
    n, m = a.shape[0], b.shape[0]
    full = _scores(eng, a, b)
    for r0, r1, c0, c1 in ((1, 34, 5, 38), (31, n, 0, m), (n - 40, n, m - 65, m), (0, 1, 0, m), (0, n, m - 1, m),
                           (17, 18, 32, 33)):
        r0, c0 = max(r0, 0), max(c0, 0)
        sub = _scores(eng, a[r0:r1], b[c0:c1])
        assert np.array_equal(sub.view(np.uint32), full[r0:r1, c0:c1].view(np.uint32)), (r0, r1, c0, c1)
    rng = np.random.default_rng(n + m)
    for i, j in [(0, 0), (n - 1, m - 1), (31, 32), (32, 31)] + list(zip(rng.integers(0, n, 12), rng.integers(0, m, 12))):
        i, j = min(i, n - 1), min(j, m - 1)
        one = _scores(eng, a[i:i + 1], b[j:j + 1])
        assert one.view(np.uint32)[0, 0] == full[i:i + 1, j].view(np.uint32)[0], (i, j)
    # repeated rows give identical cosines, whichever tile they land in
    idx = np.random.default_rng(7).integers(0, min(n, 20), 300)
    rep = _scores(eng, a[idx], b)
    assert np.array_equal(rep.view(np.uint32), full[idx].view(np.uint32))


@pytest.mark.parametrize('name', ['big_n', 'big_m'])
def test_past_one_grid_column_of_tiles(eng, name):
    """n = 65535 * 32 + 1 query rows (the last tile row is the second one its CTAs walk), or as many enrolled rows:
    the edge rows score as they do in a 1 x m call, and two calls are bit-identical."""
    case = sc.CASE_BY_NAME[name]
    a, b = sc.make(case)
    t1 = eng.cosine_scores(a, b)
    t2 = eng.cosine_scores(a, b)
    assert torch.equal(t1, t2)
    got = t1.cpu().numpy()
    if name == 'big_n':
        for i0 in (0, 65535 * 32 - 32, 65535 * 32 - 1, 65535 * 32):
            sub = _scores(eng, a[i0:i0 + 32], b)
            assert np.array_equal(sub.view(np.uint32), got[i0:i0 + 32].view(np.uint32)), i0
    else:
        for j0 in (0, 65535 * 32, case['m'] - 1):
            sub = _scores(eng, a, b[j0:j0 + 32])
            assert np.array_equal(sub.view(np.uint32), got[:, j0:j0 + 32].view(np.uint32)), j0


@pytest.mark.parametrize('name', ['shape_257x257', 'zero_self', 'scale_b_2^56'])
def test_two_calls_are_bit_identical(eng, name):
    a, b = sc.make(sc.CASE_BY_NAME[name])
    assert torch.equal(eng.cosine_scores(a, b), eng.cosine_scores(a, b))


# ------------------------------------------------------------------------------------------------ through the callers
@pytest.mark.parametrize('n,zero', [(300, (0, 150, 299)), (33, (32,))])
def test_laplacian_with_a_zero_embedding(eng, n, zero):
    """vp_spectral_laplacian starts with the kernel: a zero chunk embedding is an isolated node, as in the host path,
    instead of NaN throughout the Laplacian."""
    X = _clustered(n, seed=n)
    X[list(zero)] = 0
    _check_laplacian(eng, X)
    got = eng.spectral_laplacian(X, osp.n_drop(n)).cpu().numpy()
    host = osp.laplacian(osp.prune(osp.cosine(X), osp.n_drop(n)))
    assert np.isfinite(got).all()
    assert not got[list(zero)].any() and not got[:, list(zero)].any()
    assert not host[list(zero)].any() and not host[:, list(zero)].any()


def test_evaluate_sized_scores_with_zero_embeddings(eng):
    """An evaluate-sized trial x enrol matrix with one zero trial and one zero enrolment embedding: no score is NaN, the
    zero rows score 0, and the device metrics equal the stable host mirror on the same scores."""
    rng = np.random.RandomState(7)
    n, D, spk = 4096, 192, 400
    cen = rng.randn(spk, D)
    tl, el = rng.randint(0, spk, n).astype(np.int32), rng.randint(0, spk, n).astype(np.int32)
    trials = (cen[tl] + 1.5 * rng.randn(n, D)).astype(np.float32)
    enroll = (cen[el] + 1.5 * rng.randn(n, D)).astype(np.float32)
    trials[123] = 0
    enroll[4000] = 0
    S = eng.cosine_scores(trials, enroll)
    Sh = S.cpu().numpy()
    assert not np.isnan(Sh).any() and not Sh[123].any() and not Sh[:, 4000].any()
    got = eng.verification_metrics(S.reshape(-1), trial_labels=tl, enroll_labels=el)
    want = _host_stable_triple(Sh.reshape(-1), om.matrix_labels(tl, el))
    assert got == want
