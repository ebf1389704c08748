"""Per-element error bounds for the op-level kernel tests (tests/test_gpu_op_edges.py, tests/test_gpu_tc16_wide.py on the
GPU, tests/test_error_bound_cpu.py on the CPU).  Never imported by the product.

``BoundSim`` runs a program like plan_sim.Sim and carries, next to every fp64 value, a per-element fp64 bound beta on
|GPU - fp64|, propagated op by op from the fp32 arithmetic of the kernel that runs the op (the engine each conv resolves
to, the tensor-core kernels' K step, K block and accumulation-chunk schedule, op_cases.tc_schedule).  The bound is
computed from the case's own fp32 inputs and weight blob, never from a GPU output, so a kernel that loses part of its
work shows as an element above its own bound, however small that element is next to the largest output.

The arithmetic model (u = 2^-24, one fp32 round-to-nearest operation):
  * split TF32 operand x = hi + lo, hi = cvt.rna.tf32(x), lo read by the tensor core as TF32 (low 13 bits dropped):
    |x - hi - tf32(lo)| <= 2^-21 |x| (+ |lo| < 2^-126 where lo may be a subnormal the tensor core flushes, |x| < 2^-114),
    |lo| <= 2^-11 |x|;
  * fp16 split of x scaled by 2^s: |x - (hi + lo) 2^-s| <= max(2^-22 |x|, 2^-25 2^-s), |lo| 2^-s <= max(2^-11 |x|,
    2^-25 2^-s), with s the DESIGN exponent (amax 2^s in [2^13, 2^14), design_scale_exp: no clamp, so a kernel whose
    clamp bites is above its bound); the weight image's 2^k from the op's tc16_descale;
  * each product's split error: |a_lo w_lo| + |a - a_read| |w_hi| + |a_hi| |w - w_read|;
  * each tensor-core accumulate (three per K step of 8 (TF32) / 16 (fp16)) truncates its fp32 result and aligns its
    products to the largest addend: 2^-23 (|acc in| + |acc out|) per update, plus 2^-23 sum |a||w| per K step for the
    products themselves; accumulation chunks restart from zero and fold into the running sum with one rounding each;
  * FFMA: one rounding per fmaf, u |partial sum| along the kernel's own K order (linear_small_m: 32 lane chains and a
    5-level butterfly);
  * epilogue, glue kernels: one rounding per fp32 operation (an fma contracted by the compiler rounds less, so the
    bound stays a bound), activations add their Lipschitz constant times the incoming bound plus the CUDA Math API ulp
    bound of expf / tanhf (2 ulp each; the build has no fast-math flags); input error propagates as |W| beta_in;
  * copies, padding and max pooling are exact.
Every buffer the interpreter stores is rounded to fp32 as the GPU's is, which adds u |v| to the stored bound."""
import numpy as np

import op_cases as oc
from mvector import _lib as L
from plan_sim import Sim, _act

U = 2.0 ** -24
TRUNC = 2.0 ** -23
TF32_RHO, TF32_LAM, TF32_FLUSH = 2.0 ** -21, 2.0 ** -11, 2.0 ** -126
F16_RHO, F16_LAM, F16_FLOOR = 2.0 ** -22, 2.0 ** -11, 2.0 ** -25
ELEMS = 1 << 22                      # working-set target (fp64 elements) of one row block


def kernel_scale_exp(amax, lo=-114, hi=126):
    """common.cuh f16_scale_exp on an fp32 maximum: 13 - floor(log2 amax), clamped to [lo, hi]; 0 for 0 / inf / NaN."""
    a = np.float32(amax)
    if a == 0 or not np.isfinite(a):
        return 0
    be = int((np.array(a, dtype=np.float32).view(np.uint32) >> 23) & 0xff)
    s = 13 - (be - 127)
    return max(lo, min(hi, s))


def design_scale_exp(amax):
    """The exponent the fp16 split is designed around: amax 2^s in [2^13, 2^14), no clamp.  Taken from amax (1 + 2^-8),
    so that a GPU maximum a few ulp above the interpreter's, across a power of two, cannot give a smaller bound."""
    if amax == 0 or not np.isfinite(amax):
        return 0
    return 13 - int(np.floor(np.log2(float(amax) * (1 + 2.0 ** -8))))


def tf32_split_bounds(x):
    """-> (rho, lam): |x - hi - tf32(lo)| and |lo| bounds of the split-TF32 operand x (fp64 array)."""
    a = np.abs(x)
    flush = np.where(a < 2.0 ** -114, np.minimum(TF32_LAM * a, TF32_FLUSH), 0.0)
    return TF32_RHO * a + flush, TF32_LAM * a


def f16_split_bounds(x, s):
    """-> (rho, lam) of the fp16 split of x * 2^s, in x's units."""
    a = np.abs(x)
    floor = F16_FLOOR * 2.0 ** -s
    return np.maximum(F16_RHO * a, floor), np.maximum(F16_LAM * a, floor)


def act_bound(v, b, act):
    """Value and bound after an activation: Lipschitz constant x incoming bound + the activation's own rounding."""
    y = _act(v, act)
    if act in (L.ACT_RELU, L.ACT_HARDTANH20) or act == L.ACT_NONE:
        return y, b
    if act == L.ACT_SIGMOID:             # 1 / (1 + expf(-v)): expf 2 ulp, an add and a division
        return y, 0.25 * b + 2.0 ** -21 * np.abs(y)
    if act == L.ACT_TANH:                # tanhf: 2 ulp
        return y, b + 2.0 ** -22 * np.abs(y)
    if act == L.ACT_SILU:                # v / (1 + expf(-v)): |silu'| <= 1.1
        return y, 1.1 * b + 2.0 ** -21 * np.abs(y)
    raise ValueError(act)


def chain_abs(A, W, step, group=1):
    """Sequential accumulation of sum_k A[:, k] W[:, k], one partial sum per ``step`` columns: -> (an upper bound on the
    sum over all partials of |partial| [r, N], the final sum [r, N]).  The partials are computed (in fp32: this is a
    bound, and fp32's error is far below the 2^-10 margin applied) at the end of every ``group`` steps; a partial inside
    a group is within the group's |products| of both ends, so |P_j| <= (|P_start| + |P_end| + sum_group |p|) / 2."""
    r, K = A.shape
    N = W.shape[0]
    blk = step * group
    nb = -(-K // blk)
    if nb * blk != K:
        A = np.pad(A, ((0, 0), (0, nb * blk - K)))
        W = np.pad(W, ((0, 0), (0, nb * blk - K)))
    Ar = A.astype(np.float32).reshape(r, nb, blk).transpose(1, 0, 2)
    Wr = W.astype(np.float32).reshape(N, nb, blk).transpose(1, 2, 0)
    ends = np.zeros((r, N), dtype=np.float32)                 # sum over blocks of |P_end|
    starts = np.zeros((r, N), dtype=np.float32)               # sum over blocks of |P_start|
    P = np.zeros((r, N), dtype=np.float32)
    per = max(1, ELEMS // (r * N))
    for j0 in range(0, nb, per):
        T = np.matmul(Ar[j0:j0 + per], Wr[j0:j0 + per])
        T[0] += P
        np.cumsum(T, axis=0, out=T)
        a = np.abs(T)
        ends += a.sum(0)
        starts += a.sum(0) - a[-1] + np.abs(P)
        P = T[-1].copy()
    S = ends.astype(np.float64)
    if group > 1:
        S = S + (group - 1) / 2 * (starts + ends + np.abs(A) @ np.abs(W).T)
    return S * (1 + 2.0 ** -10), P.astype(np.float64)


def ffma_chain_bound(A, W, o):
    """u x sum |partial| of the FFMA kernels' accumulation order (conv_ffma.cu): linear_small_m's 32 lane chains (lane l
    takes k = 128 j + 4 l .. + 3) and its xor butterfly; every other FFMA kernel runs k in order."""
    if oc.kernel_of(o, L.ENGINE_FFMA) == 'linear_small_m':
        r, K = A.shape
        Kp = -(-K // 128) * 128
        Ap = np.pad(A, ((0, 0), (0, Kp - K))).reshape(r, Kp // 128, 32, 4)
        Wp = np.pad(W, ((0, 0), (0, Kp - K))).reshape(W.shape[0], Kp // 128, 32, 4)
        tot = 0.0
        lane_sums = []
        for ln in range(32):
            a, w = Ap[:, :, ln].reshape(r, -1), Wp[:, :, ln].reshape(W.shape[0], -1)
            S, _ = chain_abs(a, w, 1, 4)
            tot = tot + S
            lane_sums.append(a @ w.T)
        g = np.stack(lane_sums)                                   # [32, r, N]
        while g.shape[0] > 1:                                      # butterfly levels: groups of 2, 4, ..., 32 lanes
            g = g[0::2] + g[1::2]
            tot = tot + np.abs(g).sum(0)
        return U * tot
    S, _ = chain_abs(A, W, 1, 16)
    return U * S


def tc_acc_bound(A, W, o, engine):
    """Truncating accumulation of a tensor-core conv: 2^-23 (sum over updates of |acc in| + |acc out|) in the kernel's K
    order (K step 8 / 16, three updates per step, accumulation chunks of tc_schedule's kc K blocks restarting from zero),
    2^-23 x 4 sum |a||w| for the updates' products, and u |running sum| for every chunk fold."""
    step, bke = (16, 64) if engine == L.ENGINE_TC16 else (8, 32)
    sch = oc.tc_schedule(o, engine)
    K = A.shape[1]
    chunk = sch['kc'] * bke
    tot = 4 * (np.abs(A) @ np.abs(W).T)
    run = 0.0
    fold = 0.0
    for c, k0 in enumerate(range(0, K, chunk)):
        S, Pn = chain_abs(A[:, k0:k0 + chunk], W[:, k0:k0 + chunk], step, 4)
        Pn = np.abs(Pn)
        # per step j: updates (P_{j-1} + ..), (.. + ..), -> P_j; |in| + |out| <= 5 |P_{j-1}| + |P_j| (the lo terms'
        # contributions inside a step are in the 4 sum |a||w| above); P_0 = 0
        tot = tot + 6 * S - 5 * Pn
        run = run + A[:, k0:k0 + chunk] @ W[:, k0:k0 + chunk].T
        if c > 0:
            fold = fold + np.abs(run)
    return TRUNC * tot + U * fold


def split_bound(A, W, o, engine, s):
    """sum over k of the split error of a_k w_k (see the module docstring)."""
    aA, aW = np.abs(A), np.abs(W)
    c = 1 + 2.0 ** -10
    if engine == L.ENGINE_TC:
        rA, lA = tf32_split_bounds(A)
        rW, lW = tf32_split_bounds(W)
    else:
        k = -int(round(np.log2(o.tc16_descale)))
        rA, lA = f16_split_bounds(A, s)
        rW, lW = f16_split_bounds(W, k)
    return lA @ lW.T + c * (rA @ aW.T + aA @ rW.T)


class BoundSim(Sim):
    """plan_sim.Sim carrying a per-element bound on |GPU - fp64| next to every value.  ``engines``: the resolved engine of
    every op (op_cases.engine_of / program_engines); ``mutate``: see test_error_bound_cpu.py (None here)."""

    def __init__(self, pb, blob, feats, engines=None):
        super().__init__(pb, blob, feats)
        self.bws = np.zeros(self.ws.size)
        self.bout = np.zeros(self.out.size)
        self.binp = np.zeros(self.inp.size)
        ops = pb.finalize().ops if engines is None else None
        self.engines = engines if engines is not None else [oc.engine_of(op) for op in ops]

    def _bmem(self, off):
        if off == L.BUF_INPUT:
            return self.binp, 0
        if off == L.BUF_OUTPUT:
            return self.bout, 0
        return self.bws, off // 4

    def rdb(self, off, rows, ld, coff, C):
        mem, base = self._bmem(off)
        return mem[base + (np.arange(rows)[:, None] * ld + coff + np.arange(C)[None, :])]

    def wr(self, off, rows, ld, coff, C, val, beta=None, exact=False):
        super().wr(off, rows, ld, coff, C, val)
        mem, base = self._bmem(off)
        b = np.zeros(val.shape) if beta is None else beta
        mem[base + (np.arange(rows)[:, None] * ld + coff + np.arange(C)[None, :])] = b if exact else b + U * np.abs(val)

    def run(self):
        for self.i, o in enumerate(self.pb.ops):
            {L.OP_CONV: self.conv, L.OP_CONV_C1: self.conv, L.OP_COLSTATS: self.colstats,
             L.OP_ASP_POOL: self.asp, L.OP_EW: self.ew, L.OP_POOL2D: self.pool2d}[o.kind](o)
        assert not np.isnan(self.out).any(), 'program output not fully written'
        return self.out.copy(), self.bout.copy()

    # ------------------------------------------------------------------
    def _operand(self, o):
        """The conv's gathered source map [rows_in, cin_tot] and its bound (the add / prologue rounded once)."""
        X = self.rd(o.src, o.B * o.Tin * o.Fin, o.in_ld, o.in_coff, o.Cin)
        bX = self.rdb(o.src, o.B * o.Tin * o.Fin, o.in_ld, o.in_coff, o.Cin)
        rows_in = o.B * o.Tin * o.Fin
        if o.src2_mode == L.SRC2_ADD:
            X = X + self.rd(o.src2, rows_in, o.src2_ld, o.src2_coff, o.Cin)
            bX = bX + self.rdb(o.src2, rows_in, o.src2_ld, o.src2_coff, o.Cin) + U * np.abs(X)
        elif o.src2_mode == L.SRC2_CONCAT:
            X = np.concatenate([X, self.rd(o.src2, rows_in, o.src2_ld, o.src2_coff, o.Cin2)], axis=1)
            bX = np.concatenate([bX, self.rdb(o.src2, rows_in, o.src2_ld, o.src2_coff, o.Cin2)], axis=1)
        if o.pre_s >= 0:
            cin_tot = X.shape[1]
            s = self.w(o.pre_s, cin_tot)[None]
            X = X * s + self.w(o.pre_h, cin_tot)[None]
            bX = np.abs(s) * bX + U * np.abs(X)
            if o.pre_relu:
                X = np.maximum(X, 0)
        return X, bX

    def _im2col(self, X, bX, o, m, taps=None):
        """Rows m of the implicit-GEMM operand [len(m), K] (K ordered (tap, ci)) and its bound; padding is exact 0."""
        b = m // (o.Tout * o.Fout)
        to = (m // o.Fout) % o.Tout
        fo = m % o.Fout
        A, bA = [], []
        for kt in range(o.KT):
            for kf in range(o.KF):
                if taps is not None and kt * o.KF + kf not in taps:
                    continue
                ti = to * o.sT - o.padT + kt * o.dT
                fi = fo * o.sF - o.padF + kf * o.dF
                if o.pad_mode == L.PAD_REFLECT:
                    ti = np.where(ti < 0, -ti, ti)
                    ti = np.where(ti >= o.Tin, 2 * (o.Tin - 1) - ti, ti)
                ok = ((ti >= 0) & (ti < o.Tin) & (fi >= 0) & (fi < o.Fin))[:, None]
                row = (b * o.Tin + np.clip(ti, 0, o.Tin - 1)) * o.Fin + np.clip(fi, 0, o.Fin - 1)
                A.append(X[row] * ok)
                bA.append(bX[row] * ok)
        return np.concatenate(A, 1), np.concatenate(bA, 1)

    def conv(self, o):
        eng = self.engines[self.i] if o.kind == L.OP_CONV else L.ENGINE_FFMA
        M = o.B * o.Tout * o.Fout
        X, bX = self._operand(o)
        K = o.KT * o.KF * X.shape[1]
        W = self.wmat(o.w, o.Cout, o.w_ld, K)
        s = design_scale_exp(np.abs(X).max()) if eng == L.ENGINE_TC16 else 0
        acc = np.zeros((M, o.Cout))
        for t in range(o.KT * o.KF):                               # the value exactly as Sim.conv sums it: tap by tap
            A, _ = self._im2col(X, bX, o, np.arange(M), taps=[t])
            acc += A @ W[:, t * X.shape[1]:(t + 1) * X.shape[1]].T
        bacc = np.zeros((M, o.Cout))
        rb = max(1, min(M, ELEMS // max(K, o.Cout * 8)))
        aW = np.abs(W)
        for r0 in range(0, M, rb):
            m = np.arange(r0, min(M, r0 + rb))
            A, bA = self._im2col(X, bX, o, m)
            b = bA @ aW.T
            if eng in (L.ENGINE_TC, L.ENGINE_TC16):
                b += split_bound(A, W, o, eng, s) + tc_acc_bound(A, W, o, eng)
            else:
                b += ffma_chain_bound(A, W, o)
            bacc[m] = b
        self._epilogue(o, eng, acc, bacc)

    def _epilogue(self, o, eng, v, b):
        M = o.B * o.Tout * o.Fout
        m = np.arange(M)
        seg = np.minimum(((m // o.Fout) % o.Tout) // o.seg_len, o.n_seg - 1)
        urow = m // (o.Tout * o.Fout) * o.n_seg + seg
        if o.bias >= 0:
            v = v + self.w(o.bias, o.Cout)[None]
        if o.bias >= 0 or eng == L.ENGINE_TC16:          # acc + bias (tensor cores: fmaf(acc, descale, bias))
            b = b + U * np.abs(v)
        if o.ubias != L.BUF_NONE:
            v = v + self.rd(o.ubias, o.B * o.n_seg, o.Cout, 0, o.Cout)[urow]
            b = b + self.rdb(o.ubias, o.B * o.n_seg, o.Cout, 0, o.Cout)[urow] + U * np.abs(v)
        v, b = act_bound(v, b, o.act)
        if o.post_s >= 0:
            ps = self.w(o.post_s, o.Cout)[None]
            v = v * ps + self.w(o.post_h, o.Cout)[None]
            b = np.abs(ps) * b + U * np.abs(v)
        if o.gate != L.BUF_NONE:
            g = self.rd(o.gate, o.B * o.n_seg, o.Cout, 0, o.Cout)[urow]
            bg = self.rdb(o.gate, o.B * o.n_seg, o.Cout, 0, o.Cout)[urow]
            b = np.abs(g) * b + np.abs(v) * bg
            v = v * g
            b = b + U * np.abs(v)
        if o.res != L.BUF_NONE:
            v = v + self.rd(o.res, M, o.res_ld, o.res_coff, o.Cout)
            b = b + self.rdb(o.res, M, o.res_ld, o.res_coff, o.Cout) + U * np.abs(v)
        v, b = act_bound(v, b, o.act2)
        self.wr(o.dst, M, o.out_ld, o.out_coff, o.Cout, v, b)
        if o.sum != L.BUF_NONE:
            sv = self.rd(o.sum, M, o.sum_ld, o.sum_coff, o.Cout) + v
            sb = self.rdb(o.sum, M, o.sum_ld, o.sum_coff, o.Cout) + b + U * np.abs(sv)
            self.wr(o.sum, M, o.sum_ld, o.sum_coff, o.Cout, sv, sb)

    # ---- glue kernels (pool.cu) ----
    @staticmethod
    def _warp_sum(T, bT):
        """Sum over axis 1 of [B, R, C] as pool.cu does it: 8 warp chains (rows w, w + 8, ...), then warp 0 adds the
        eight totals in order.  -> (sum [B, C], bound)."""
        B, R, C = T.shape
        Rp = -(-R // 8) * 8
        Tp = np.pad(T, ((0, 0), (0, Rp - R), (0, 0))).reshape(B, Rp // 8, 8, C)
        P = np.cumsum(Tp, axis=1)
        chains = U * np.abs(P).sum(1).sum(1)
        pre = np.cumsum(P[:, -1], axis=1)
        return pre[:, -1], bT.sum(1) + chains + U * np.abs(pre[:, 1:]).sum(1)

    def colstats(self, o):
        R = o.Tin * o.Fin
        X = self.rd(o.src, o.B * R, o.in_ld, o.in_coff, o.Cin).reshape(o.B, R, o.Cin)
        bX = self.rdb(o.src, o.B * R, o.in_ld, o.in_coff, o.Cin).reshape(o.B, R, o.Cin)
        tot, btot = self._warp_sum(X, bX)
        if o.mode == L.STATS_SEG_CONTEXT:
            segs = [self._warp_sum(X[:, s * o.seg_len:(s + 1) * o.seg_len], bX[:, s * o.seg_len:(s + 1) * o.seg_len])
                    for s in range(o.n_seg)]
            if o.n_seg <= 64:                  # total = segment sums added in order
                acc = np.cumsum(np.stack([s for s, _ in segs]), axis=0)
                tot = acc[-1]
                btot = sum(b for _, b in segs) + U * np.abs(acc[1:]).sum(0)
            mean = tot / R
            bmean = btot / R + U * np.abs(mean)
            out = np.zeros((o.B, o.n_seg, o.Cin))
            bout = np.zeros_like(out)
            for s, (ss, bss) in enumerate(segs):
                cnt = min(o.seg_len, R - s * o.seg_len)
                q = ss / cnt
                out[:, s] = mean + q
                bout[:, s] = bmean + bss / cnt + U * np.abs(q) + U * np.abs(out[:, s])
            self.wr(o.dst, o.B * o.n_seg, o.out_ld, o.out_coff, o.Cin, out.reshape(-1, o.Cin), bout.reshape(-1, o.Cin))
            return
        mean = tot / R
        bmean = btot / R + U * np.abs(mean)
        if o.mode == L.STATS_MEAN:
            self.wr(o.dst, o.B, o.out_ld, o.out_coff, o.Cin, mean, bmean)
            return
        d = X - mean[:, None]
        bd = bX + bmean[:, None] + U * np.abs(d)
        ssq, bssq = self._warp_sum(d * d, 2 * np.abs(d) * bd + bd * bd)     # fmaf(d, d, q): the chain's roundings
        if o.mode == L.STATS_MEAN_VAR_UNBIASED:
            sd = ssq / (R - 1)
            bsd = bssq / (R - 1) + U * sd
        else:
            t = ssq / (R if o.mode == L.STATS_MEAN_STD_CLAMP else R - 1)
            bt = bssq / (R if o.mode == L.STATS_MEAN_STD_CLAMP else R - 1) + U * t
            if o.mode == L.STATS_MEAN_STD_CLAMP:
                bt = np.where(t + bt <= o.eps, 0.0, bt)
                t = np.maximum(t, o.eps)
            elif o.mode == L.STATS_MEAN_STD_TSTP:
                t = t + o.eps
                bt = bt + U * t
            sd = np.sqrt(t)
            bsd = bt / (sd + np.sqrt(np.maximum(t - bt, 0))) + U * sd
        self.wr(o.dst, o.B, o.out_ld, o.out_coff, 2 * o.Cin, np.concatenate([mean, sd], 1),
                np.concatenate([bmean, bsd], 1))

    def asp(self, o):
        T, Cn = o.Tin, o.Cin
        X = self.rd(o.src, o.B * T, o.in_ld, o.in_coff, Cn).reshape(o.B, T, Cn)
        bX = self.rdb(o.src, o.B * T, o.in_ld, o.in_coff, Cn).reshape(o.B, T, Cn)
        Lg = self.rd(o.src2, o.B * T, o.src2_ld, o.src2_coff, Cn).reshape(o.B, T, Cn)
        bL = self.rdb(o.src2, o.B * T, o.src2_ld, o.src2_coff, Cn).reshape(o.B, T, Cn)
        z = Lg - Lg.max(1, keepdims=True)
        dz = U * np.abs(z) + bL + bL.max(1, keepdims=True)
        e = np.exp(z)
        be = e * (1.01 * dz + 2.0 ** -22)                         # expf: 2 ulp; dz << 1
        se, bse = self._warp_sum(e, be)
        sx, bsx = self._warp_sum(e * X, be * np.abs(X) + e * bX)
        mean = sx / se
        bmean = (bsx + np.abs(mean) * bse) / (se - bse) + U * np.abs(mean)
        if o.mode == 1:
            self.wr(o.dst, o.B, o.out_ld, o.out_coff, Cn, mean, bmean)
            return
        d = X - mean[:, None]
        bd = bX + bmean[:, None] + U * np.abs(d)
        dd = d * d
        bdd = 2 * np.abs(d) * bd + bd * bd + U * dd
        sq, bsq = self._warp_sum(e * dd, be * dd + e * bdd)
        t = sq / se
        bt = (bsq + t * bse) / (se - bse) + U * t
        bt = np.where(t + bt <= o.eps, 0.0, bt)
        t = np.maximum(t, o.eps)
        sd = np.sqrt(t)
        bsd = bt / (sd + np.sqrt(np.maximum(t - bt, 0))) + U * sd
        self.wr(o.dst, o.B, o.out_ld, o.out_coff, 2 * Cn, np.concatenate([mean, sd], 1), np.concatenate([bmean, bsd], 1))

    def pool2d(self, o):
        X = self.rd(o.src, o.B * o.Tin * o.Fin, o.in_ld, o.in_coff, o.Cin).reshape(o.B, o.Tin, o.Fin, o.Cin)
        bX = self.rdb(o.src, o.B * o.Tin * o.Fin, o.in_ld, o.in_coff, o.Cin).reshape(o.B, o.Tin, o.Fin, o.Cin)
        out = np.zeros((o.B, o.Tout, o.Fout, o.Cin))
        bout = np.zeros_like(out)
        n = o.KT * o.KF
        for to in range(o.Tout):
            for fo in range(o.Fout):
                t0, f0 = to * o.sT - o.padT, fo * o.sF - o.padF
                win = X[:, max(t0, 0):min(t0 + o.KT, o.Tin), max(f0, 0):min(f0 + o.KF, o.Fin)]
                bw = bX[:, max(t0, 0):min(t0 + o.KT, o.Tin), max(f0, 0):min(f0 + o.KF, o.Fin)]
                if o.mode == 0:
                    out[:, to, fo] = win.max(axis=(1, 2))
                    bout[:, to, fo] = bw.max(axis=(1, 2))
                    continue
                part = np.cumsum(win.reshape(o.B, -1, o.Cin), axis=1)
                out[:, to, fo] = part[:, -1] / n
                # the in-order sum, then x fl(1 / n): two more roundings
                bout[:, to, fo] = ((bw.reshape(o.B, -1, o.Cin).sum(1) + U * np.abs(part[:, 1:]).sum(1)) / n
                                   + 2 * U * np.abs(out[:, to, fo]))
        self.wr(o.dst, o.B * o.Tout * o.Fout, o.out_ld, o.out_coff, o.Cin, out.reshape(-1, o.Cin),
                bout.reshape(-1, o.Cin), exact=o.mode == 0)

    def ew(self, o):
        rpu = o.Tin * o.Fin
        rows = o.B * rpu
        v = self.rd(o.src, rows, o.in_ld, o.in_coff, o.Cin)
        b = self.rdb(o.src, rows, o.in_ld, o.in_coff, o.Cin)
        if o.mode == L.EW_PAD_COPY:
            self.wr(o.dst, rows, o.out_ld, o.out_coff, o.Cout, np.pad(v, ((0, 0), (0, o.Cout - o.Cin))),
                    np.pad(b, ((0, 0), (0, o.Cout - o.Cin))), exact=True)
            return
        if o.mode == L.EW_GATE_RES:
            if o.gate != L.BUF_NONE:
                u = np.arange(rows) // rpu
                g = self.rd(o.gate, o.B, o.Cin, 0, o.Cin)[u]
                b = np.abs(g) * b + np.abs(v) * self.rdb(o.gate, o.B, o.Cin, 0, o.Cin)[u]
                v = v * g
                b = b + U * np.abs(v)
            if o.res != L.BUF_NONE:
                v = v + self.rd(o.res, rows, o.res_ld, o.res_coff, o.Cin)
                b = b + self.rdb(o.res, rows, o.res_ld, o.res_coff, o.Cin) + U * np.abs(v)
            v, b = act_bound(v, b, o.act2)
        elif o.mode == L.EW_AFF:
            y = self.rd(o.src2, rows, o.src2_ld, o.src2_coff, o.Cin)
            by = self.rdb(o.src2, rows, o.src2_ld, o.src2_coff, o.Cin)
            t = np.tanh(self.rd(o.res, rows, o.res_ld, o.res_coff, o.Cin))
            bt = self.rdb(o.res, rows, o.res_ld, o.res_coff, o.Cin) + 2.0 ** -22 * np.abs(t)
            a = 1 + t
            ba = bt + U * np.abs(a)
            c = 2 - a
            bc = ba + U * np.abs(c)
            p1, p2 = v * a, y * c
            b = (np.abs(a) * b + np.abs(v) * ba + U * np.abs(p1) + np.abs(c) * by + np.abs(y) * bc + U * np.abs(p2))
            v = p1 + p2
            b = b + U * np.abs(v)
        else:                                                     # EW_COPY
            self.wr(o.dst, rows, o.out_ld, o.out_coff, o.Cin, v, b, exact=True)
            return
        self.wr(o.dst, rows, o.out_ld, o.out_coff, o.Cin, v, b)


_CACHE = {}


def bounded(b, key=None, engines=None):
    """-> (fp64 reference, per-element bound), both [out_rows, out_cols], of a Built case (op_cases.build).  ``key``: a
    name to cache the pair under (the bound of a long-K case takes seconds)."""
    if key is not None and key in _CACHE:
        return _CACHE[key]
    ref, beta = BoundSim(b.pb, b.blob, b.X, engines).run()
    r = ref.reshape(b.out_rows, b.out_cols), beta.reshape(b.out_rows, b.out_cols)
    if key is not None:
        _CACHE[key] = r
    return r


def ratio(got, ref, beta):
    """max |got - ref| / beta elementwise; an element with beta = 0 must be equal (else inf); NaN / inf in got -> inf."""
    d = np.abs(got.astype(np.float64) - ref)
    if not np.isfinite(d).all():
        return float('inf')
    r = np.where(beta > 0, d / np.where(beta > 0, beta, 1.0), np.where(d > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def max_rel(got, ref, floor=1.0):
    """The flat metric the gates used before: max |got - ref| / max(floor, max |ref|)."""
    return float(np.abs(got.astype(np.float64) - ref).max() / max(floor, np.abs(ref).max()))
