"""Case table, fp64 oracle and per-element error bound for the op-level tests of the cosine score kernel
(csrc/pool.cu cosine_scores_kernel, ABI vp_cosine_scores): tests/test_gpu_cosine_scores.py on the GPU,
tests/test_score_cases_cpu.py on the CPU.  Never imported by the product.

The kernel (launch_cosine_scores): one CTA of 256 threads per 32 x 32 tile of scores, grid (ceil(m / 32),
min(ceil(n / 32), 65535)); the CTAs of one grid row walk the tile rows with a stride of gridDim.y.  A tile stages its 32
a rows and 32 b rows through shared memory in K chunks of 64 columns, zero-filled past n, m and D.  A thread holds one
column j and four rows i and keeps dot = <a_i, b_j>, |a_i|^2 and |b_j|^2 as one fmaf chain each over k = 0 .. D-1 (the
zero fill adds exact zeros), then writes dot / (sqrtf(|a_i|^2) sqrtf(|b_j|^2)) with a zero norm taken as 1.

``plan`` restates that launch arithmetic; every case records the launch or data edge it is meant to reach (``intent``)
and the CPU suite checks that it does.

Oracle (``cosine64``): sklearn's cosine_similarity in fp64 -- normalise every row, a zero row to the zero vector, then
one product -- so a zero-norm row scores 0 against everything.  (sklearn's normalize also leaves a row whose norm is
below 10 eps of its dtype unnormalised; neither the oracle nor the kernel does that: both are scale invariant down to
an exact zero.)  A row holding a NaN makes its whole row or column NaN.

Error bound (``bound``; u = 2^-24, every fp32 operation rounds to nearest with gradual underflow: the build has no
fast-math flags, so sqrtf and '/' are correctly rounded).  With s = sum_k a_k b_k, t = sum_k |a_k b_k|, p = |a|^2,
q = |b|^2 over the fp32 inputs, exactly, and r = s / sqrt(pq):
  1. A chain of D fmaf rounds each partial sum once, so every term carries at most D factors (1 + delta), |delta| <= u,
     and each step may add one subnormal rounding error <= eta = 2^-150:
         |dot - s| <= gamma_D t + 2 D eta,   gamma_D = D u / (1 - D u),
     and likewise |na - p| <= gamma_D p + 2 D eta, |nb - q| <= gamma_D q + 2 D eta.
  2. With eps_p = (gamma_D p + 2 D eta) / p, sqrt(na) = sqrt(p) (1 + phi_p), |phi_p| <= eps_p / (2 - eps_p), since
     |sqrt(1 + e) - 1| = |e| / (1 + sqrt(1 + e)).
  3. The denominator fl(fl(sqrt na) fl(sqrt nb)) = sqrt(pq) (1 + theta), |theta| <= theta_max =
     (1 + phi_p)(1 + phi_q)(1 + u)^3 - 1: two square roots and one product, each rounded once.
  4. The division rounds once more:  score = (s + e)(1 + delta) / (sqrt(pq)(1 + theta)), so
         |score - r| <= beta = [(1 + u)(gamma_D t + 2 D eta) / sqrt(pq) + (u + theta_max) |r|] / (1 - theta_max).
By Cauchy-Schwarz t <= sqrt(pq) and |r| <= 1, so beta <= (2 gamma_D + 4 u)(1 + O(gamma_D)) whatever the magnitudes of the
operands: 3.6e-7 at D = 1, 2.3e-5 at D = 192, 6.1e-5 at D = 512.  Where the dot product cancels (t >> |s|) beta stays
gamma_D t / sqrt(pq), the error the chain can really make there.  A pair with a zero row gets beta = 0: the kernel's dot
is then a sum of signed zeros starting from +0, exactly +0, and so is the score.
The bound is evaluated in fp64 from the inputs; the fp64 sums and the oracle's r err by less than (D + 2) 2^-53 (t /
sqrt(pq) + |r|), under 2^-28 of beta, which the factor (1 + 2^-10) covers.
Scope: every nonzero row has 2^-126 <= p < 2^127, so no norm, square root or denominator leaves fp32's normal range.
Past it the reference's own float32 normalisation fails as well."""
import zlib

import numpy as np

U = 2.0 ** -24
ETA = 2.0 ** -150
TILE, K_CHUNK, GRID_Y_MAX = 32, 64, 65535
NORMAL_MIN, SUMSQ_MAX = 2.0 ** -126, 2.0 ** 127
INT_BIG = 65535 * 32 + 1                       # 2,097,121: the first row count whose tile rows exceed one grid column


# ---------------------------------------------------------------------------------------------------------------
# launch arithmetic (launch_cosine_scores, pool.cu)
# ---------------------------------------------------------------------------------------------------------------
def plan(n, m, D):
    """-> the launch of one n x m x D call: grid, tile counts, rows / columns / K columns in the last tile and chunk,
    and how many tile rows the busiest CTA walks."""
    row_tiles, col_tiles, k_chunks = -(-n // TILE), -(-m // TILE), -(-D // K_CHUNK)
    gy = min(row_tiles, GRID_Y_MAX)
    return dict(grid=(col_tiles, gy), row_tiles=row_tiles, col_tiles=col_tiles,
                row_tail=n - TILE * (row_tiles - 1), col_tail=m - TILE * (col_tiles - 1),
                k_chunks=k_chunks, k_tail=D - K_CHUNK * (k_chunks - 1), row_passes=-(-row_tiles // gy))


# ---------------------------------------------------------------------------------------------------------------
# oracle and bound
# ---------------------------------------------------------------------------------------------------------------
def _nan_rows(x):
    return np.isnan(x).any(axis=1)


def cosine64(a, b):
    """fp64 cosine matrix [n, m] with sklearn's zero convention; NaN on the rows / columns of rows holding a NaN."""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    na, nb = np.linalg.norm(a64, axis=1), np.linalg.norm(b64, axis=1)
    an = a64 / np.where(na == 0, 1.0, na)[:, None]
    bn = b64 / np.where(nb == 0, 1.0, nb)[:, None]
    r = np.nan_to_num(an) @ np.nan_to_num(bn).T
    r[_nan_rows(a64), :] = np.nan
    r[:, _nan_rows(b64)] = np.nan
    return r


def gamma(D):
    return D * U / (1 - D * U)


def bound(a, b, r=None):
    """Per-element bound beta [n, m] on |kernel - cosine64| (module docstring); 0 where a row is zero, NaN where the
    oracle is NaN."""
    a64, b64 = np.asarray(a, np.float64), np.asarray(b, np.float64)
    D = a64.shape[1]
    r = cosine64(a, b) if r is None else r
    g, tail = gamma(D), 2 * D * ETA
    p, q = (a64 * a64).sum(axis=1), (b64 * b64).sum(axis=1)
    t = np.abs(a64) @ np.abs(b64).T
    with np.errstate(divide='ignore', invalid='ignore'):
        ep, eq = (g * p + tail) / p, (g * q + tail) / q
        phi_p, phi_q = ep / (2 - ep), eq / (2 - eq)
        theta = (1 + phi_p)[:, None] * (1 + phi_q)[None, :] * (1 + U) ** 3 - 1
        pq = np.sqrt(p)[:, None] * np.sqrt(q)[None, :]
        beta = ((1 + U) * (g * t + tail) / pq + (U + theta) * np.abs(r)) / (1 - theta) * (1 + 2.0 ** -10)
    beta[p == 0, :] = 0.0
    beta[:, q == 0] = 0.0
    beta[np.isnan(r)] = np.nan
    return beta


def check(got, a, b):
    """Assert got [n, m] (fp32) is the cosine matrix of a, b within the bound: NaN exactly where the oracle has NaN, an
    exact zero where a row is zero, |got - oracle| <= beta elsewhere.  -> the worst err / beta."""
    r = cosine64(a, b)
    beta = bound(a, b, r)
    got = np.asarray(got)
    assert got.shape == r.shape and got.dtype == np.float32, (got.shape, got.dtype)
    nan = np.isnan(r)
    bad = np.argwhere(np.isnan(got) != nan)
    assert not bad.size, f'{len(bad)} elements NaN where the oracle is not, or not NaN where it is: {bad[:4].tolist()}'
    exact = ~nan & (beta == 0)
    bad = np.argwhere(exact & (got != 0))
    assert not bad.size, f'{len(bad)} scores of a zero-norm row are not 0: {bad[:4].tolist()}'
    rest = ~nan & ~exact
    err = np.abs(got[rest].astype(np.float64) - r[rest])
    worst = float((err / beta[rest]).max()) if err.size else 0.0
    if worst > 1:
        idx = np.argwhere(rest)[np.argmax(err / beta[rest])]
        raise AssertionError(f'err / beta = {worst:.3g} at {tuple(idx)}: got {got[tuple(idx)]!r}, '
                             f'fp64 {r[tuple(idx)]!r}, beta {beta[tuple(idx)]:.3g}')
    return worst


def fp32_sequential(a, b, mutation=None):
    """A plain float32 evaluation in numpy with the kernel's summation order and zero rule: each product and each
    partial sum rounded on its own (no fma), then sqrt, product and quotient.  ``mutation`` makes it wrong on purpose:
    'drop_last_k' leaves out column D-1 (a K chunk that overflows by one, lost), 'tf32' reads the operands with a
    10-bit mantissa."""
    a32, b32 = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if mutation == 'tf32':
        a32, b32 = ((x.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32) for x in (a32, b32))
    D = a32.shape[1] - (1 if mutation == 'drop_last_k' else 0)
    dot = np.zeros((a32.shape[0], b32.shape[0]), np.float32)
    na, nb = np.zeros(a32.shape[0], np.float32), np.zeros(b32.shape[0], np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        for k in range(D):
            ak, bk = a32[:, k], b32[:, k]
            dot += ak[:, None] * bk[None, :]
            na += ak * ak
            nb += bk * bk
        ra = np.where(na == 0, np.float32(1), np.sqrt(na))
        rb = np.where(nb == 0, np.float32(1), np.sqrt(nb))
        return dot / (ra[:, None] * rb[None, :])


# ---------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------
SHAPES = (1, 31, 32, 33, 63, 64, 65, 257)
# n -> (tile rows, rows in the last tile), by hand
TILES = {1: (1, 1), 31: (1, 31), 32: (1, 32), 33: (2, 1), 63: (2, 31), 64: (2, 32), 65: (3, 1), 257: (9, 1)}
# D -> (K chunks, columns in the last chunk), by hand
K_CHUNKS = {1: (1, 1), 3: (1, 3), 4: (1, 4), 63: (1, 63), 64: (1, 64), 65: (2, 1), 127: (2, 63), 128: (2, 64),
            129: (3, 1), 192: (3, 64), 512: (8, 64)}
SCALES = (-60, -40, -20, 20, 40, 56)


def _case(name, n, m, D, data='gauss', intent=None, **kw):
    return dict(name=name, n=n, m=m, D=D, data=data, intent=dict(intent or {}), seed=zlib.crc32(name.encode()), **kw)


def _shape_intent(n, m):
    (rt, rtail), (ct, ctail) = TILES[n], TILES[m]
    return dict(row_tiles=rt, row_tail=rtail, col_tiles=ct, col_tail=ctail)


def _k_intent(D):
    kc, kt = K_CHUNKS[D]
    return dict(k_chunks=kc, k_tail=kt)


CASES = (
    # every partial / full / one-past last tile row against every such last tile column
    [_case(f'shape_{n}x{m}', n, m, 192, intent=_shape_intent(n, m)) for n in SHAPES for m in SHAPES]
    # K chunks that are partial, exact, or overflow by one column
    + [_case(f'k_D{D}', 65, 33, D, intent=dict(_k_intent(D), row_tail=1, col_tail=1)) for D in K_CHUNKS]
    # |cos| within 1e-6 of 1, both signs: column j is a scaled, slightly perturbed copy of row j mod n
    + [_case(f'parallel_D{D}', 33, 65, D, 'parallel', intent=_k_intent(D)) for D in (65, 192, 512)]
    # near-orthogonal pairs with components up to 1e6: the dot product cancels
    + [_case(f'orthogonal_D{D}', 33, 65, D, 'orthogonal', intent=_k_intent(D)) for D in (65, 192, 512)]
    # a 10^9 dynamic range inside every row
    + [_case(f'range_D{D}', 33, 65, D, 'range', intent=_k_intent(D)) for D in (65, 192, 512)]
    # one operand scaled by 2^e: 512 unit-size components keep the fp32 sum of squares normal and finite
    + [_case(f'scale_{w}_2^{e}', 33, 65, 512, 'scale', intent=_k_intent(512), which=w, exp=e)
       for w in ('a', 'b') for e in SCALES]
    # zero rows in a, in b, in both, and in X against X; rows on both sides of a tile edge
    + [_case('zero_a', 65, 33, 192, 'zero', za=(0, 31, 32, 64), zb=()),
       _case('zero_b', 33, 65, 192, 'zero', za=(), zb=(0, 31, 32, 64)),
       _case('zero_both', 65, 65, 129, 'zero', za=(1, 32, 64), zb=(0, 33, 64)),
       _case('zero_1x1', 1, 1, 192, 'zero', za=(0,), zb=(0,)),
       _case('zero_self', 65, 65, 192, 'self', za=(5, 32, 64)),
       _case('zero_self_D3', 33, 33, 3, 'self', za=(0, 32))]
    # one NaN row in each operand, next to full tiles of healthy rows
    + [_case('nan_rows', 65, 65, 192, 'nan', nan_a=(33,), nan_b=(31,))]
    # past one grid column of tile rows, and 2^16 tile columns
    + [_case('big_n', INT_BIG, 3, 4, intent=dict(grid=(1, GRID_Y_MAX), row_passes=2, row_tail=1, k_tail=4)),
       _case('big_m', 3, INT_BIG, 4, intent=dict(grid=(INT_BIG // TILE + 1, 1), row_passes=1, col_tail=1))]
)
CASE_BY_NAME = {c['name']: c for c in CASES}


def make(case):
    """-> (a [n, D], b [m, D]) float32, C-contiguous; b is a itself for 'self' cases."""
    n, m, D, kind = case['n'], case['m'], case['D'], case['data']
    rng = np.random.default_rng(case['seed'])
    if kind in ('gauss', 'zero', 'self', 'nan', 'scale'):
        a, b = rng.standard_normal((n, D)), rng.standard_normal((m, D))
        if kind == 'scale':
            if case['which'] == 'a':
                a = a * 2.0 ** case['exp']
            else:
                b = b * 2.0 ** case['exp']
        if kind in ('zero', 'self'):
            a[list(case['za']), :] = 0
        if kind == 'zero':
            b[list(case['zb']), :] = 0
        if kind == 'nan':
            a[list(case['nan_a']), D // 2] = np.nan
            b[list(case['nan_b']), D - 1] = np.nan
    elif kind == 'parallel':
        a = rng.standard_normal((n, D))
        b = np.empty((m, D))
        for j in range(m):
            base = a[j % n].astype(np.float32).astype(np.float64)
            delta = 1e-4 * (j % 3) * rng.standard_normal(D) * np.abs(base).mean()
            b[j] = (-1) ** j * 2.0 ** (j % 5 - 2) * (base + delta)
    elif kind == 'orthogonal':
        big = rng.choice(D, size=min(4, D), replace=False)
        a = rng.standard_normal((n, D)) * 1e3
        a[:, big] *= 1e3
        a = a.astype(np.float32).astype(np.float64)
        g = rng.standard_normal((m, D)) * 1e3
        g[:, big] *= 1e3
        b = np.empty((m, D))
        for j in range(m):
            u = a[j % n] / np.linalg.norm(a[j % n])
            b[j] = g[j] - (g[j] @ u) * u
    elif kind == 'range':
        def rows(k):
            x = 10.0 ** rng.uniform(-9, 0, (k, D)) * rng.choice([-1.0, 1.0], (k, D))
            for i in range(k):
                lo, hi = rng.choice(D, size=2, replace=False)
                x[i, lo], x[i, hi] = np.sign(x[i, lo]) * 1e-9, np.sign(x[i, hi])
            return x
        a, b = rows(n), rows(m)
    else:
        raise ValueError(kind)
    a = np.ascontiguousarray(a, np.float32)
    return (a, a) if kind == 'self' else (a, np.ascontiguousarray(b, np.float32))


def zero_rows(case):
    """-> (zero rows of a, zero rows of b) the case plants."""
    if case['data'] == 'zero':
        return tuple(case['za']), tuple(case['zb'])
    if case['data'] == 'self':
        return tuple(case['za']), tuple(case['za'])
    return (), ()
