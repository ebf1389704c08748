"""CPU side of the cosine score cases (tests/score_cases.py): every case reaches the launch or data edge its intent names,
the table covers each edge, the fp64 oracle agrees with the host cosines and sklearn, and the a-priori bound holds for a
plain float32 evaluation while the same evaluation made subtly wrong exceeds it."""
import numpy as np
import pytest

import score_cases as sc
from oracle import spectral as osp


def _ids(c):
    return c['name']


@pytest.mark.parametrize('case', sc.CASES, ids=_ids)
def test_case_reaches_its_launch_edge(case):
    p = sc.plan(case['n'], case['m'], case['D'])
    for k, v in case['intent'].items():
        assert p[k] == v, (k, p[k], v)
    gx, gy = p['grid']
    assert 1 <= gx < 2 ** 31 and 1 <= gy <= 65535
    assert (p['row_passes'] - 1) * gy < p['row_tiles'] <= p['row_passes'] * gy


def test_table_covers_every_edge():
    plans = [sc.plan(c['n'], c['m'], c['D']) for c in sc.CASES]
    shapes = {(c['n'], c['m']) for c in sc.CASES if c['name'].startswith('shape_')}
    assert shapes == {(n, m) for n in sc.SHAPES for m in sc.SHAPES}
    for key in ('row_tail', 'col_tail'):                         # last tile partial by 31 / 1, full, one past
        assert {1, 31, 32} <= {p[key] for p in plans}, key
    assert {1, 2, 3, 9} <= {p['row_tiles'] for p in plans} and {1, 2, 3, 9} <= {p['col_tiles'] for p in plans}
    assert {c['D'] for c in sc.CASES} >= set(sc.K_CHUNKS)
    assert {(p['k_chunks'], p['k_tail']) for p in plans} >= {(1, 1), (1, 63), (1, 64), (2, 1), (2, 63), (2, 64),
                                                             (3, 1), (8, 64)}
    assert any(c['D'] % 4 for c in sc.CASES)                     # the kernel takes any D
    assert max(p['row_passes'] for p in plans) == 2              # a CTA walks a second tile row
    assert max(p['grid'][0] for p in plans) > 65535              # tile columns past gridDim.y's limit
    big = [c for c in sc.CASES if max(c['n'], c['m']) > 65535 * 32]
    assert {(c['n'] > c['m']) for c in big} == {True, False}
    kinds = {c['data'] for c in sc.CASES}
    assert kinds >= {'gauss', 'parallel', 'orthogonal', 'range', 'scale', 'zero', 'self', 'nan'}
    sw = {(c['which'], c['exp']) for c in sc.CASES if c['data'] == 'scale'}
    assert {('a', -60), ('a', 56), ('b', -60), ('b', 56)} <= sw
    za = [sc.zero_rows(c) for c in sc.CASES]
    assert any(a and not b for a, b in za) and any(b and not a for a, b in za) and any(a and b for a, b in za)


@pytest.mark.parametrize('case', sc.CASES, ids=_ids)
def test_case_data_has_its_property(case):
    a, b = sc.make(case)
    n, m, D = case['n'], case['m'], case['D']
    assert a.shape == (n, D) and b.shape == (m, D) and a.dtype == b.dtype == np.float32
    assert a.flags.c_contiguous and b.flags.c_contiguous
    za, zb = sc.zero_rows(case)
    nan_a, nan_b = np.isnan(a).any(axis=1), np.isnan(b).any(axis=1)
    # every other row lies in the bound's scope: its fp32 sum of squares is normal and finite
    for x, z, bad in ((a, za, nan_a), (b, zb, nan_b)):
        p = (x.astype(np.float64) ** 2).sum(axis=1)
        live = ~bad
        live[list(z)] = False
        assert (p[list(z)] == 0).all()
        assert (p[live] >= sc.NORMAL_MIN).all() and (p[live] < sc.SUMSQ_MAX).all()
    kind = case['data']
    if kind in ('parallel', 'orthogonal'):
        r = sc.cosine64(a, b)
        paired = r[np.arange(m) % n, np.arange(m)]
        t = np.abs(a.astype(np.float64)) @ np.abs(b.astype(np.float64)).T
        t /= np.linalg.norm(a.astype(np.float64), axis=1)[:, None] * np.linalg.norm(b.astype(np.float64), axis=1)
        if kind == 'parallel':
            assert (np.abs(paired) >= 1 - 1e-6).all() and (paired > 0).any() and (paired < 0).any()
            assert (np.abs(paired) < 1).any()                     # perturbed copies, not only exact multiples
        else:
            # the dot product cancels: the sum of |a_k b_k| is at least 10^4 times the sum of a_k b_k
            assert (np.abs(paired) <= 1e-6).all() and (t[np.arange(m) % n, np.arange(m)] >= 1e4 * np.abs(paired)).all()
            assert np.abs(a).max() >= 1e5 and np.abs(b).max() >= 1e5
    elif kind == 'range':
        for x in (a, b):
            ax = np.abs(x.astype(np.float64))
            assert (ax.max(axis=1) / ax.min(axis=1) >= 1e9 * (1 - 1e-6)).all()
    elif kind == 'scale':
        x = a if case['which'] == 'a' else b
        mx = np.abs(x).max(axis=1).astype(np.float64) * 2.0 ** -case['exp']
        assert (mx > 0.5).all() and (mx < 8).all()               # unit-size components times 2^e
    elif kind in ('zero', 'self'):
        assert not a[list(za)].any() and not b[list(zb)].any()
        if kind == 'self':
            assert b is a
    elif kind == 'nan':
        assert list(np.flatnonzero(nan_a)) == list(case['nan_a']) and list(np.flatnonzero(nan_b)) == list(case['nan_b'])
        assert np.isnan(a).sum() == len(case['nan_a']) and np.isnan(b).sum() == len(case['nan_b'])


def _sklearn_scope(x):
    """sklearn's normalize also leaves a row whose norm is below 10 eps unnormalised; compare only where no row is in
    that band."""
    nrm = np.linalg.norm(x.astype(np.float64), axis=1)
    return ((nrm == 0) | (nrm >= 10 * np.finfo(np.float64).eps)).all()


@pytest.mark.parametrize('case', [c for c in sc.CASES if c['data'] != 'nan' and c['n'] + c['m'] < 4096], ids=_ids)
def test_oracle_matches_host_cosines(case):
    """The fp64 oracle against the float32 host cosine of the diarization path (oracle/spectral.cosine, the form of
    SpectralCluster.get_sim_mat, on the stacked rows of a and b), which must lie within the bound as well, and against
    sklearn's cosine_similarity in fp64, zeros included.  sklearn refuses NaN input."""
    from sklearn.metrics.pairwise import cosine_similarity
    a, b = sc.make(case)
    n = case['n']
    r = sc.cosine64(a, b)
    beta = sc.bound(a, b, r)
    host = osp.cosine(a) if b is a else osp.cosine(np.vstack([a, b]))[:n, n:]
    za, zb = sc.zero_rows(case)
    assert not host[list(za)].any() and not host[:, list(zb)].any()
    assert not r[list(za)].any() and not r[:, list(zb)].any()
    assert (np.abs(host.astype(np.float64) - r) <= beta).all()
    if _sklearn_scope(a) and _sklearn_scope(b):
        sk = cosine_similarity(a.astype(np.float64), b.astype(np.float64))
        assert not sk[list(za)].any() and not sk[:, list(zb)].any()
        assert np.abs(sk - r).max() <= 1e-13


@pytest.mark.parametrize('case', sc.CASES, ids=_ids)
def test_bound_holds_for_plain_fp32(case):
    """An honest float32 kernel stays within beta, so the bound is not tighter than fp32 arithmetic allows.  Its products
    and partial sums round separately, which still gives every term at most D roundings: the first addition, to 0, is
    exact.  Zero rows score exactly 0, NaN stays in its own
    row and column."""
    a, b = sc.make(case)
    got = sc.fp32_sequential(a, b)
    worst = sc.check(got, a, b)
    print(f"{case['name']}: plain fp32 err / beta {worst:.3f}")


@pytest.mark.parametrize('name,mutation', [('k_D65', 'drop_last_k'), ('k_D129', 'drop_last_k'), ('k_D3', 'drop_last_k'),
                                           ('shape_257x257', 'drop_last_k'), ('big_n', 'drop_last_k'),
                                           ('k_D129', 'tf32'), ('shape_257x257', 'tf32'), ('parallel_D512', 'tf32'),
                                           ('orthogonal_D192', 'tf32'), ('scale_a_2^-60', 'tf32')])
def test_bound_catches_mutations(name, mutation):
    """The same evaluation made subtly wrong -- one K column lost from the last chunk, or operands read as TF32 -- has
    an element above its bound."""
    a, b = sc.make(sc.CASE_BY_NAME[name])
    with pytest.raises(AssertionError, match='err / beta'):
        sc.check(sc.fp32_sequential(a, b, mutation), a, b)


def test_zero_rule_is_checked():
    """check() insists on an exact 0 for a zero row; the unguarded 0 / 0 of a kernel without the zero rule is NaN."""
    case = sc.CASE_BY_NAME['zero_self']
    a, b = sc.make(case)
    got = sc.fp32_sequential(a, b)
    z = list(case['za'])
    assert not got[z].any() and not got[:, z].any() and not np.signbit(got[z]).any()
    bad = got.copy()
    bad[z[0], z[0]] = np.nan
    with pytest.raises(AssertionError):
        sc.check(bad, a, b)
    bad = got.copy()
    bad[z[1], 3] = np.float32(1e-30)
    with pytest.raises(AssertionError):
        sc.check(bad, a, b)


def test_bound_is_magnitude_free():
    """beta <= (2 gamma_D + 4 u)(1 + 2^-8) in every case, and scaling an operand by 2^e changes it only through the
    underflow term 2 D eta / |a|^2, which reaches 2^-14 of beta at 2^-60."""
    for c in sc.CASES:
        a, b = sc.make(c)
        beta = sc.bound(a, b)
        cap = (2 * sc.gamma(c['D']) + 4 * sc.U) * (1 + 2.0 ** -8)
        assert np.nanmax(beta) <= cap, (c['name'], np.nanmax(beta), cap)
        if c['data'] == 'scale':
            s = np.float32(2.0 ** -c['exp'])
            a1, b1 = (a * s, b) if c['which'] == 'a' else (a, b * s)
            assert np.allclose(sc.bound(a1, b1), beta, rtol=2.0 ** -13, atol=0), c['name']
