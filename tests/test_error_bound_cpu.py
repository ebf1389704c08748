"""CPU checks of the per-element error bounds (tests/error_bound.py) that gate the op-level GPU tests.

(a) The split residual bounds hold on a large sample of fp32 bit patterns, fp16-subnormal lo terms and both ends of the
    fp16 split's scale range included.
(b) A numpy emulation of the kernels' arithmetic -- split TF32 (cvt.rna hi, lo read as TF32, three truncating fp32
    accumulates per K8 step, accumulation chunks folded with round-to-nearest adds), the fp16 split (power-of-two
    activation scale from the kernel's f16_scale_exp, K16 steps, the pack_tc16 weight image) and the FFMA kernels' fp32
    fmaf chains in their own K order -- stays within the bound on the geometries of named op cases: K tails, chunk
    remainders, one-row M tails, N tails, the wide fp16-split kernel's K tails and its range cases.  Rows are reduced to
    the last 64 of each case (its M tail).
(c) The same emulation with each kernel mutation the bound must catch exceeds it on the case that names it: lo lost on
    each tile's last K block (M1), on the last M tile (M2), the A_hi B_lo MMA skipped on one K step of four (M3), lo
    lost on the wide kernel's last K block (M4), the activation scale exponent clamped to +-100 (M5)."""
import numpy as np
import pytest

import error_bound as eb
import op_cases as oc
from mvector import _lib as L
from mvector.engine import tf32_rna

TABLE = {**oc.TC_CASES, **oc.ENGINE_CASES, **oc.FFMA_CASES, **oc.TC16_WIDE_CASES}


# ---------------------------------------------------------------------------------------------------------------
# (a) split residuals
# ---------------------------------------------------------------------------------------------------------------
def _bits(rng, n, lo_exp, hi_exp):
    """n random fp32 values with exponents in [lo_exp, hi_exp] and uniform random mantissa bits, random signs."""
    e = rng.integers(lo_exp + 127, hi_exp + 128, n).astype(np.uint32)
    m = rng.integers(0, 1 << 23, n).astype(np.uint32)
    s = rng.integers(0, 2, n).astype(np.uint32)
    return ((s << 31) | (e << 23) | m).view(np.float32)


def _tf32_trunc(x):
    """What the tensor core reads of an fp32 operand in TF32 mode: the low 13 mantissa bits dropped."""
    return (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def _f16_split(x32, s):
    """publish() / split_f16: xs = x 2^s in fp32, hi = fp16(xs), lo = fp16(xs - hi) -> (hi, lo) as fp32 values."""
    with np.errstate(over='ignore', invalid='ignore'):
        xs = (x32 * np.float32(2.0 ** s)).astype(np.float32)
        hi = xs.astype(np.float16).astype(np.float32)
        lo = (xs - hi).astype(np.float16).astype(np.float32)
    return hi, lo


def test_tf32_split_residual_bound():
    rng = np.random.default_rng(1)
    # every normal exponent except the top one, where cvt.rna can round up to inf; the lo term is subnormal below 2^-115
    x = _bits(rng, 1 << 20, -126, 126)
    hi = tf32_rna(x)
    lo = (x - hi).astype(np.float32)
    got = np.abs(x.astype(np.float64) - hi - _tf32_trunc(lo))
    rho, lam = eb.tf32_split_bounds(x.astype(np.float64))
    assert (got <= rho).all() and (np.abs(lo) <= lam).all()
    print(f'tf32 split: max residual / bound {np.max(got / rho):.3f}, max |lo| / bound {np.max(np.abs(lo) / lam):.3f}')


@pytest.mark.parametrize('amax_exp', [-113, -60, -1, 0, 40, 127])
def test_f16_split_residual_bound(amax_exp):
    """x over 40 binades below a slot maximum 2^amax_exp (fp16-subnormal lo and hi terms included), split at the
    kernel's scale exponent, which equals the design exponent over the whole range the split supports."""
    rng = np.random.default_rng(amax_exp + 200)
    amax = np.float32(2.0 ** amax_exp * 1.75)
    s = eb.kernel_scale_exp(amax)
    assert s == eb.design_scale_exp(amax) == 13 - amax_exp
    x = _bits(rng, 1 << 20, max(-126, amax_exp - 40), amax_exp)
    hi, lo = _f16_split(x, s)
    got = np.abs(x.astype(np.float64) - (hi.astype(np.float64) + lo) * 2.0 ** -s)
    rho, lam = eb.f16_split_bounds(x.astype(np.float64), s)
    assert np.isfinite(hi).all() and (got <= rho).all() and (np.abs(lo) * 2.0 ** -s <= lam).all()
    sub = np.abs(lo) < 2.0 ** -14
    assert sub.any()                                              # fp16-subnormal lo terms are in the sample
    print(f'f16 split at 2^{amax_exp}: max residual / bound {np.max(got / rho):.3f} '
          f'({sub.mean():.1%} subnormal lo terms)')


def test_f16_scale_exp_clamp():
    """The kernel's exponent is the design exponent from 2^-113 to the largest float; the old +-100 clamp is not."""
    for e in (-113, -87, 0, 86, 116, 127):
        amax = np.float32(2.0 ** e)
        assert eb.kernel_scale_exp(amax) == eb.design_scale_exp(amax) == 13 - e
    assert eb.kernel_scale_exp(np.float32(np.finfo(np.float32).max)) == -114
    assert eb.kernel_scale_exp(np.float32(2.0 ** -120)) == 126                  # below the supported range
    assert eb.kernel_scale_exp(np.float32(2.0 ** 116), -100, 100) != 13 - 116
    assert eb.kernel_scale_exp(np.float32(2.0 ** -110), -100, 100) != 13 + 110


# ---------------------------------------------------------------------------------------------------------------
# (b), (c) emulated kernels against the bound
# ---------------------------------------------------------------------------------------------------------------
def _trunc32(x):
    """fp64 -> fp32 rounded toward zero (a truncating tensor-core accumulate), back in fp64."""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f.astype(np.float64)


def _rn32(x):
    return x.astype(np.float32).astype(np.float64)


class Gemm:
    """The implicit GEMM of a case's conv on its last ``rows`` output rows: A [rows, K], W [N, K] (fp32 values in
    fp64), the op, its engine, the rows' indices and the bound of the accumulator."""

    def __init__(self, name, rows=64, **over):
        case = dict(TABLE[name], **over)
        b = oc.build(case)
        self.o = o = b.pb.finalize().ops[b.main]
        self.engine = b.expect[b.main] if o.kind == L.OP_CONV else L.ENGINE_FFMA
        s = eb.BoundSim(b.pb, b.blob, b.X)
        for s.i, op in enumerate(b.pb.ops[:b.main]):               # the copies that feed the op
            {L.OP_EW: s.ew}[op.kind](op)
        X, _ = s._operand(o, s.reader(o), np.arange(o.B * o.Tin * o.Fin))
        M = o.B * o.Tout * o.Fout
        self.m = np.arange(max(0, M - rows), M)
        self.A, _ = s._im2col(X, np.zeros_like(X), o, self.m)
        self.W = s.wmat(o.w, o.Cout, o.w_ld, self.A.shape[1])
        self.amax = np.float32(np.abs(X).max())
        self.s = eb.design_scale_exp(self.amax)
        self.exact = self.A @ self.W.T
        if self.engine in (L.ENGINE_TC, L.ENGINE_TC16):
            self.beta = (eb.split_bound(self.A, self.W, o, self.engine, self.s)
                         + eb.tc_acc_bound(self.A, self.W, o, self.engine))
        else:
            self.beta = eb.ffma_chain_bound(self.A, self.W, o)

    def emulate(self, mutate=None):
        if self.engine == L.ENGINE_FFMA:
            return _emulate_ffma(self)
        return _emulate_tc(self, mutate)

    def ratio(self, got):
        return eb.ratio(got, self.exact, self.beta)

    def flat(self, got):
        return eb.max_rel(got, self.exact)


def _emulate_tc(g, mutate):
    o, tc16 = g.o, g.engine == L.ENGINE_TC16
    A32, W32 = g.A.astype(np.float32), g.W.astype(np.float32)
    K = A32.shape[1]
    step, bke = (16, 64) if tc16 else (8, 32)
    sch = oc.tc_schedule(o, g.engine)
    if tc16:
        s = eb.kernel_scale_exp(g.amax, *((-100, 100) if mutate == 'M5' else (-114, 126)))
        k = -int(round(np.log2(o.tc16_descale)))
        Ah, Al = _f16_split(A32, s)
        Wh, Wl = _f16_split(W32, k)
        descale = 2.0 ** (-s - k)
    else:
        Ah = tf32_rna(A32)
        Al = _tf32_trunc((A32 - Ah).astype(np.float32))
        Wh = tf32_rna(W32)
        Wl = _tf32_trunc((W32 - Wh).astype(np.float32))
        descale = 1.0
    Ah, Al, Wh, Wl = (v.astype(np.float64) for v in (Ah, Al, Wh, Wl))
    kblocks = -(-K // bke)
    if mutate in ('M1', 'M4'):                       # lo = 0 on each tile's last K block
        Al[:, (kblocks - 1) * bke:] = 0
    if mutate == 'M2':                               # lo = 0 on the rows of the last M tile
        Al[g.m >= (sch['m_tiles'] - 1) * 128] = 0
    chunk = sch['kc'] * bke
    run = None
    with np.errstate(over='ignore', invalid='ignore'):
        for k0 in range(0, K, chunk):
            acc = np.zeros_like(g.exact)
            for j0 in range(k0, min(K, k0 + chunk), step):
                c = slice(j0, j0 + step)
                acc = _trunc32(acc + Al[:, c] @ Wh[:, c].T)
                if not (mutate == 'M3' and (j0 // step) % 4 == 3):      # kk = 3 of the K block
                    acc = _trunc32(acc + Ah[:, c] @ Wl[:, c].T)
                acc = _trunc32(acc + Ah[:, c] @ Wh[:, c].T)
            run = acc if run is None else _rn32(acc + run)
        return run * descale


def _emulate_ffma(g):
    A, W = g.A, g.W
    if oc.kernel_of(g.o, L.ENGINE_FFMA) == 'linear_small_m':
        K = A.shape[1]
        Kp = -(-K // 128) * 128
        Ap = np.pad(A, ((0, 0), (0, Kp - K))).reshape(len(A), Kp // 128, 32, 4)
        Wp = np.pad(W, ((0, 0), (0, Kp - K))).reshape(len(W), Kp // 128, 32, 4)
        lanes = []
        for ln in range(32):
            acc = np.zeros_like(g.exact)
            for j in range(Kp // 128):
                for i in range(4):
                    acc = _rn32(acc + np.outer(Ap[:, j, ln, i], Wp[:, j, ln, i]))
            lanes.append(acc)
        v = np.stack(lanes)
        while len(v) > 1:                          # xor butterfly: the pairs a lane adds hold the same group sums
            v = _rn32(v[0::2] + v[1::2])
        return v[0]
    acc = np.zeros_like(g.exact)
    for k in range(A.shape[1]):
        acc = _rn32(acc + np.outer(A[:, k], W[:, k]))
    return acc


# the bound's healthy geometries: K tails (K = 4, 12, 72, 120), N tails (20, 196, 192), one-row M tails, chunk
# remainders (K = 576 by 256, 1600 by 512), the longest unchunked K (1536), a chunked K = 4096, the wide kernel's K tails
# and one partial K block, its range cases, and the FFMA kernels (tiled with a K tail, small-M at K = 3072)
HEALTHY = ['k4_1x1-tc', 'k12_k3_cin4-tc', 'k72_1x1-tc', 'k72_1x1-tc16', 'k120_k3_cin40-tc16', 'm_tail1_n20-tc',
           'm_tail1_n196-tc16', 'eres_k576-tc', 'eres_k576-tc16', 'default_k1600-tc', 'default_k1600-tc16',
           'gemm_k1536_n128_ubias_tanh-tc', 'gemm_k1536_n128_ubias_tanh-tc16', 'n_tail_192-tc16',
           'long_k_chunked_4096_n128-tc', 'k_tail_72-tc', 'k_tail_72-ffma', 'k_tail', 'k_tail_136',
           'k8_one_partial_block', 'scale_2^-110', 'scale_2^116', 'tiled_m2049_n68', 'small_m_m1023_k3072_n192_ubias']

# mutation -> the cases it must fail on (every one of them): short K blocks, a chunk remainder, the one-row M tail, a
# K tail of the wide kernel and the wide kernel's range cases past the old clamp
MUTATIONS = {
    'M1': ['k72_1x1-tc', 'eres_k576-tc', 'k120_k3_cin40-tc16', 'k72_1x1-tc16'],
    'M2': ['m_tail1_n20-tc', 'm_tail1_n196-tc16'],
    'M3': ['k72_1x1-tc', 'eres_k576-tc', 'k72_1x1-tc16', 'default_k1600-tc16'],
    'M4': ['k_tail', 'k_tail_136'],
    'M5': ['scale_2^-110', 'scale_2^116'],
}


@pytest.fixture(scope='module')
def gemms():
    return {n: Gemm(n) for n in sorted(set(HEALTHY).union(*MUTATIONS.values()))}


def test_healthy_emulation_within_bound(gemms):
    worst = {}
    for n in HEALTHY:
        g = gemms[n]
        got = g.emulate()
        r = g.ratio(got)
        print(f'{n}: err/beta {r:.3f} (max-rel {g.flat(got):.2e})')
        fam = {L.ENGINE_TC: 'split TF32', L.ENGINE_TC16: 'fp16 split'}.get(g.engine, 'FFMA')
        worst[fam] = max(worst.get(fam, 0.0), r)
        assert r <= 1.0, (n, r)
    print('worst healthy err/beta: ' + ', '.join(f'{k} {v:.3f}' for k, v in worst.items()))


@pytest.mark.parametrize('mutation', list(MUTATIONS))
def test_mutations_exceed_bound(gemms, mutation):
    for n in MUTATIONS[mutation]:
        g = gemms[n]
        got = g.emulate(mutation)
        r = g.ratio(got)
        print(f'{mutation} on {n}: err/beta {r:.3g} (max-rel {g.flat(got):.2e})')
        assert r > 1.0, (mutation, n, r)
