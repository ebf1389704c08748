"""Case tables and a single-op harness for the op-level kernel tests (tests/test_gpu_op_edges.py on the GPU,
tests/test_op_edges_cpu.py on the CPU).

A case is a dict.  ``build(case)`` lowers it into a one-op (or few-op) program with PlanBuilder / WeightArena: the op
under test, the copies that feed it (a tracked workspace source for the fp16 split, gate / per-utterance-bias rows, an
accumulate-into view, the columns around an output window) and, for the amax cases, a TC16 conv consuming its output.
``run_gpu`` runs the program through Program.run_profiled; ``Sim(pb, blob, X).run()`` (tests/plan_sim.py) is the
fp64 reference.

Every case names the kernel it is meant to reach (``kernel``) and, for convs, the engine it requests (``engine``;
'auto' expects the engine ``engine_of`` resolves); the GPU tests assert the engine from run_profiled, the CPU tests
re-derive the kernel from the lowered op with the launchers' own predicates (``kernel_of``, ``tc_schedule``), so a
table entry cannot drift into covering something else.  Never imported by the product."""
import os

import numpy as np

from mvector import _lib as L
from mvector.engine import PlanBuilder, View, WeightArena, tc_tile_n

SMS = 132                                   # H100 SXM: the persistent tensor-core grid is min(SMs, tiles)
ENGINES = {'auto': L.ENGINE_AUTO, 'ffma': L.ENGINE_FFMA, 'tc': L.ENGINE_TC, 'tc16': L.ENGINE_TC16}
ERES_POLICY = (512, 256)                    # models/eres2net.py: chunk K > 512 by 256
DEFAULT_POLICY = (1536, 512)                # models/base.py


# ---------------------------------------------------------------------------------------------------------------
# harness
# ---------------------------------------------------------------------------------------------------------------
class _Inputs:
    """Column allocator over the program input [rows, width]: every tensor the program reads from outside is a column
    window of it, filled after the plan is known.  ``derived`` columns are computed from other columns (and the weight
    blob) after the random fill: the host-materialised operand of a gather twin (see ``_conv``)."""

    def __init__(self, width):
        self.width, self.used, self.rows, self.fills, self.derived = width, 0, 1, [], []

    def take(self, rows, C, fill=('normal', 1.0, 0.0), skew=0):
        c = self.used + skew
        self.used = (c + C + 3) // 4 * 4
        self.rows = max(self.rows, rows)
        self.fills.append((c, C, fill))
        return View(L.BUF_INPUT, self.width, c, C)

    def data(self, rng, scale):
        X = np.zeros((self.rows, self.width), dtype=np.float64)
        for c, C, (dist, s, shift) in self.fills:
            shape = (self.rows, C)
            if dist == 'normal':
                v = rng.standard_normal(shape) * s + shift
            elif dist == 'negative':                    # strictly negative: max pooling must not see a 0 from padding
                v = -(np.abs(rng.standard_normal(shape)) + 0.05) * s
            elif dist == 'gate':                        # gates / per-row factors stay O(1) at every input scale
                v = rng.uniform(0.5, 1.5, shape) * s
                X[:, c:c + C] = v
                continue
            elif dist == 'saturate':                    # |att| in [4, 30]: tanh is +-1 (or within an ulp of it)
                v = rng.uniform(4, 30, shape) * rng.choice([-1.0, 1.0], shape)
                X[:, c:c + C] = v
                continue
            else:
                raise ValueError(dist)
            X[:, c:c + C] = v * scale
        return X.astype(np.float32)


class Built:
    """A lowered case: pb / blob / X for Sim and Program, the output shape, which op is under test, and the engine every
    conv op must resolve to."""

    def __init__(self, case, pb, arena, X, out_rows, out_cols, main, expect, consumer=None):
        self.case, self.pb, self.arena, self.X = case, pb, arena, X
        self.blob = arena.blob()
        self.out_rows, self.out_cols = out_rows, out_cols
        self.main, self.expect, self.consumer = main, expect, consumer


def _copy(pb, src, dst, rows):
    o = pb.ew(L.EW_COPY, src, dst, rows)
    o.B = 1
    return o


def _out(pb, inp, rows, C, coff=0):
    """Program output [rows, C] or, with coff > 0, the column window [coff, coff + C) of a wider output whose other
    columns are written first by copies: a kernel that strays outside its window overwrites them."""
    if not coff:
        return pb.output_view(C, rows), C
    width = coff + C + 8
    full = pb.output_view(width, rows)
    _copy(pb, inp.take(rows, coff), full.cols(0, coff), rows)
    _copy(pb, inp.take(rows, 8), full.cols(coff + C, 8), rows)
    return full.cols(coff, C), width


def _conv(pb, arena, inp, c, rng, expect, src=None, dst=None):
    """One CONV / CONV_C1 op from a case dict.  ``src`` / ``dst``: views supplied by a writer -> consumer pair."""
    B, Tin, Fin, Cin, N = c['B'], c['Tin'], c.get('Fin', 1), c['Cin'], c['N']
    Tout, Fout = c.get('Tout', Tin), c.get('Fout', Fin)
    KT, KF = c.get('KT', 1), c.get('KF', 1)
    c1 = c.get('c1', False)
    src2_mode = c.get('src2_mode', L.SRC2_NONE)
    Cin2 = c.get('Cin2', Cin) if src2_mode != L.SRC2_NONE else 0
    cin_tot = 1 if c1 else Cin + (Cin2 if src2_mode == L.SRC2_CONCAT else 0)
    K = KT * KF * cin_tot
    rows_in, rows_out = B * Tin * Fin, B * Tout * Fout
    n_seg = c.get('n_seg', 1)
    engine = c.get('engine', 'ffma')
    in_coff = c.get('in_coff', 0)
    xfill = ('normal', c.get('xscale', 1.0), 0.0)
    src2 = None
    xcol = ycol = None                                         # input columns holding x / the added second source
    if src is not None:
        pass
    elif c1:
        inp.take(rows_in, 1, fill=xfill)                       # the one-channel map is the flat start of the input
        src = View(L.BUF_INPUT, 1, 0, 1)
    elif engine == 'tc16' and not c.get('raw_input'):
        # the fp16 split scales by the source tensor's tracked maximum: the source is a workspace tensor written by
        # program ops; with a concat, both halves are windows of ONE allocation (two writers, one amax slot).
        # ``raw_input``: read the program input itself, which has no amax slot
        a = pb.alloc(rows_in, in_coff + Cin + Cin2)
        src = a.cols(in_coff, Cin)
        _copy(pb, inp.take(rows_in, Cin, fill=xfill), src, rows_in)
        if src2_mode == L.SRC2_CONCAT:
            src2 = a.cols(in_coff + Cin, Cin2)
            _copy(pb, inp.take(rows_in, Cin2, fill=xfill), src2, rows_in)
    else:
        src = inp.take(rows_in, Cin, fill=xfill, skew=in_coff)
        xcol = src.coff
        if src2_mode != L.SRC2_NONE and c.get('src2_width'):
            # the second source in an allocation of its own (another row pitch, another first column), filled by a copy
            y = inp.take(rows_in, Cin2, fill=xfill)
            ycol = y.coff
            src2 = pb.alloc(rows_in, c['src2_width']).cols(c.get('src2_coff', 0), Cin2)
            _copy(pb, y, src2, rows_in)
        elif src2_mode != L.SRC2_NONE:
            src2 = inp.take(rows_in, Cin2, fill=xfill)
            ycol = src2.coff
    W = rng.standard_normal((N, K)) / np.sqrt(K)
    w = arena.add('w', W) if c1 else arena.add_conv('w', W)
    bias = arena.add('b', rng.standard_normal(N) * 0.1 * c.get('bias_scale', 1.0)) if c.get('bias') else -1
    post = (arena.add('ps', rng.uniform(0.5, 1.5, N)), arena.add('ph', rng.standard_normal(N) * 0.2)) if c.get('post') else None
    pre = None
    if c.get('pre'):
        # 'pow2': signed power-of-two scales, so x * s is exact and fmaf(x, s, h) == fl32(x * s + h) (see twin())
        s = (rng.choice([-1.0, 1.0], cin_tot) * 2.0 ** rng.integers(-2, 3, cin_tot) if c['pre'] == 'pow2'
             else rng.uniform(0.5, 1.5, cin_tot))
        pre = (arena.add('qs', s), arena.add('qh', rng.standard_normal(cin_tot) * 0.2))
    pre_relu = bool(pre) and c.get('pre_relu', True)
    res = inp.take(rows_out, N, fill=xfill) if c.get('res') else None
    gate = ubias = None
    if c.get('gate'):
        gate = pb.alloc(B * n_seg, N)
        _copy(pb, inp.take(B * n_seg, N, fill=('gate', 1.0, 0.0)), gate, B * n_seg)
    if c.get('ubias'):
        ubias = pb.alloc(B * n_seg, N)
        _copy(pb, inp.take(B * n_seg, N), ubias, B * n_seg)
    out_cols = None
    acc = None
    if dst is None:
        dst, out_cols = _out(pb, inp, rows_out, N * (2 if c.get('sum') else 1), c.get('out_coff', 0))
        full = dst
        dst = full.cols(0, N)
    if c.get('sum'):                     # accumulate-into view: prefilled, acc += y, then copied out next to y
        acc = pb.alloc(rows_out, N)
        _copy(pb, inp.take(rows_out, N), acc, rows_out)
    if c.get('twin'):
        # MODE 0 twin of an add / prologue conv: everything above is laid out (and drawn from the rngs) exactly as for
        # the original, and the op reads one extra input block holding the operand the original's gather computes
        assert xcol is not None and (pre is not None or src2_mode == L.SRC2_ADD), 'twin of an add / prologue conv'
        op = inp.take(rows_in, Cin)
        inp.derived.append(dict(col=op.coff, rows=rows_in, C=Cin, x=xcol, y=ycol, pre=pre, pre_relu=pre_relu))
        src, src2, src2_mode, pre, pre_relu = op, None, L.SRC2_NONE, None, False
    expect[len(pb.ops)] = ENGINES[engine] if not c1 else 0
    main = len(pb.ops)
    pb.conv(src, dst, w, K, Tin, Tout, Fin=Fin, Fout=Fout, KT=KT, KF=KF, sT=c.get('sT', 1), sF=c.get('sF', 1),
            dT=c.get('dT', 1), dF=1, padT=c.get('padT', 0), padF=c.get('padF', 0),
            pad_mode=c.get('pad_mode', L.PAD_ZERO), bias=bias, pre=pre, pre_relu=pre_relu, post=post,
            act=c.get('act', L.ACT_NONE), act2=c.get('act2', L.ACT_NONE), res=res, gate=gate, ubias=ubias,
            seg_len=c.get('seg_len'), n_seg=n_seg, src2=src2, src2_mode=src2_mode, sum_into=acc,
            engine=ENGINES[engine], c1=c1)
    if acc is not None:
        _copy(pb, acc, full.cols(N, N), rows_out)
    return main, dst, out_cols, rows_out, N


def _pool2d(pb, inp, c, dst=None):
    B, Tin, Fin, C = c['B'], c['Tin'], c['Fin'], c['C']
    k, s, pad = c.get('k', 3), c.get('stride', 1), c.get('pad', 1)
    Tout, Fout = (Tin + 2 * pad - k) // s + 1, (Fin + 2 * pad - k) // s + 1
    src = inp.take(B * Tin * Fin, C, fill=(c.get('fill', 'normal'), 1.0, 0.0), skew=c.get('in_coff', 0))
    out_cols = None
    if dst is None:
        dst, out_cols = _out(pb, inp, B * Tout * Fout, C, c.get('out_coff', 0))
    main = len(pb.ops)
    pb.pool2d(src, dst, L.POOL_MAX if c['mode'] == 'max' else L.POOL_AVG, Tin, Fin, Tout, Fout, k=k, stride=s, pad=pad)
    return main, dst, out_cols, B * Tout * Fout, C


def _ew(pb, inp, c, dst=None):
    """EW in GATE_RES / AFF / COPY / PAD_COPY mode over B utterances x T rows."""
    B, T, C = c['B'], c['T'], c['C']
    rows = B * T
    mode = getattr(L, 'EW_' + c['mode'])
    skew = c.get('in_coff', 0)
    if mode == L.EW_PAD_COPY:
        Cout = c['Cout']
        x = inp.take(rows, C, skew=skew)
        out_cols = None
        if dst is None:
            dst, out_cols = _out(pb, inp, rows, Cout, c.get('out_coff', 0))
        main = len(pb.ops)
        o = pb._new(L.OP_EW)                       # the same op PlanBuilder.input_view1d emits, on any view
        o.mode = L.EW_PAD_COPY
        o.src, o.in_ld, o.in_coff, o.Cin = x.off, x.ld, x.coff, C
        o.dst, o.out_ld, o.out_coff, o.Cout = dst.off, dst.ld, dst.coff, Cout
        o.Tin, o.Fin = T, 1
        pb._emit(o, dst=dst, src=x)
        return main, dst, out_cols, rows, Cout
    x = inp.take(rows, C, skew=skew)
    gate = res = y = att = None
    if mode == L.EW_GATE_RES:
        if c.get('gate'):
            gate = pb.alloc(B, C)
            _copy(pb, inp.take(B, C, fill=('gate', 1.0, 0.0)), gate, B)
        if c.get('res'):
            res = inp.take(rows, C, skew=skew)
    elif mode == L.EW_AFF:
        y = inp.take(rows, C, skew=skew)
        att = inp.take(rows, C, fill=('saturate', 1.0, 0.0) if c.get('saturate') else ('normal', 1.0, 0.0), skew=skew)
    out_cols = None
    if dst is None:
        dst, out_cols = _out(pb, inp, rows, C, c.get('out_coff', 0))
    main = len(pb.ops)
    pb.ew(mode, x, dst, T, gate=gate, res=res, y=y, att=att, act2=c.get('act2', L.ACT_NONE))
    return main, dst, out_cols, rows, C


def _pool(pb, inp, c):
    """COLSTATS / ASP_POOL over B utterances x R rows of C columns."""
    B, R, C = c['B'], c['R'], c['C']
    skew = c.get('in_coff', 0)
    x = inp.take(B * R, C, fill=c.get('fill', ('normal', 2.0, 0.0)), skew=skew)
    main = len(pb.ops)
    if c['op'] == 'asp':
        logits = inp.take(B * R, C, fill=('normal', 2.0, c.get('logit_shift', 0.0)), skew=skew)
        n_rows, n_cols = B, C if c.get('mean_only') else 2 * C
        pb.asp_pool(x, logits, pb.output_view(n_cols, n_rows), R, eps=1e-12, mean_only=c.get('mean_only', False))
    else:
        mode = getattr(L, 'STATS_' + c['stats'])
        seg_len = c.get('seg_len')
        n_seg = -(-R // seg_len) if seg_len else 1
        n_rows = B * n_seg
        n_cols = C if mode in (L.STATS_MEAN, L.STATS_SEG_CONTEXT) else 2 * C
        pb.colstats(x, pb.output_view(n_cols, n_rows), R, mode, eps=1e-5, seg_len=seg_len, n_seg=n_seg)
    return main, n_rows, n_cols


def _emit_op(pb, arena, inp, c, rng, expect, dst=None):
    if c['op'] in ('conv', 'c1'):
        return _conv(pb, arena, inp, dict(c, c1=c['op'] == 'c1'), rng, expect, dst=dst)
    if c['op'] == 'pool2d':
        return _pool2d(pb, inp, c, dst=dst)
    if c['op'] == 'ew':
        return _ew(pb, inp, c, dst=dst)
    raise ValueError(c['op'])


def _build(case, width):
    rng = np.random.default_rng(case['seed'])
    arena = WeightArena(*case.get('policy', DEFAULT_POLICY))
    arena.add('unused', np.zeros(4))
    inp = _Inputs(width)
    pb = PlanBuilder(case.get('B', 1), L.ENGINE_AUTO)
    expect = {}
    consumer = None
    if case['op'] in ('colstats', 'asp'):
        main, out_rows, out_cols = _pool(pb, inp, case)
    elif 'consumer' in case:
        # writer -> TC16 conv: the writer's output is a workspace allocation (or, with `windows`, several writers share
        # one allocation) that the consumer reads whole; its amax slot is the only thing that scales the fp16 split
        writers = case.get('windows', [case])
        B, rows_per_utt = case['consumer']['B'], case['consumer']['T']
        rows = B * rows_per_utt
        C = sum(w['out_C'] for w in writers)
        a = pb.alloc(rows, C)
        col = 0
        main = []
        for w in writers:
            m, _, _, r, cw = _emit_op(pb, arena, inp, w, rng, expect, dst=a.cols(col, w['out_C']))
            assert r == rows and cw == w['out_C'], (r, rows, cw)
            main.append(m)
            col += cw
        main = main[0] if len(main) == 1 else main
        cc = dict(case['consumer'], op='conv', engine='tc16', Cin=C, Tin=rows_per_utt)
        consumer, _, out_cols, out_rows, _ = _conv(pb, arena, inp, cc, rng, expect, src=a)
    else:
        main, _, out_cols, out_rows, _ = _emit_op(pb, arena, inp, case, rng, expect)
    pb.in_floats = inp.rows * width
    return pb, arena, inp, main, expect, consumer, out_rows, out_cols


def build(case):
    """Lower a case -> Built.  Two passes: the first sizes the input matrix, the second lays the plan out on it."""
    width = max(4, (_build(case, 1 << 16)[2].used + 3) // 4 * 4)
    pb, arena, inp, main, expect, consumer, out_rows, out_cols = _build(case, width)
    X = inp.data(np.random.default_rng(case['seed'] + 7919), case.get('scale', 1.0))
    for i, e in expect.items():
        if e == L.ENGINE_AUTO and pb.ops[i].kind == L.OP_CONV:
            expect[i] = engine_of(pb.finalize().ops[i])
    b = Built(case, pb, arena, X, out_rows, out_cols, main, expect, consumer)
    for d in inp.derived:
        X[:d['rows'], d['col']:d['col'] + d['C']] = _gathered(X, b.blob, d)
    return b


def _gathered(X, blob, d):
    """The A-operand map an add / prologue gather feeds the MMAs, materialised on the host in the kernels' arithmetic:
    fl32(x + y) for the add, and fmaf(x, s, h) (then max(., 0) with pre_relu) for the prologue.  With power-of-two s,
    x * s is exact and fl32(fl64(x * s) + h) is the correctly rounded fp32 sum (53 >= 2 * 24 + 2): exactly fmaf."""
    rows, C = d['rows'], d['C']
    x = X[:rows, d['x']:d['x'] + C]
    if d['pre'] is None:
        return x + X[:rows, d['y']:d['y'] + C]                                  # float32 + float32: one rounding
    s, h = (blob[o // 4:o // 4 + C].astype(np.float64) for o in d['pre'])
    assert np.array_equal(np.abs(s), 2.0 ** np.round(np.log2(np.abs(s)))), 'twin needs power-of-two prologue scales'
    v = (x.astype(np.float64) * s + h).astype(np.float32)
    return np.maximum(v, np.float32(0)) if d['pre_relu'] else v


def twin(case):
    """The MODE 0 twin of an add / prologue case: same weights blob, geometry, epilogue, tc_bn / tc_kc and engine, reading
    the host-materialised operand (``_gathered``) as a plain source.  Its output must equal the original's bit for bit:
    the tensor-core kernel shares everything after the gather (split, MMA order, epilogue) between the modes, and the FFMA
    kernel runs one gather (common.cuh gather_a4) whose add / prologue are the same fp32 operations."""
    return dict(case, twin=True)


def with_batch(case, B):
    """The same case at another batch size (every table entry lowers from B)."""
    return dict(case, B=B)


def sim(b):
    from plan_sim import Sim
    return Sim(b.pb, b.blob, b.X).run().reshape(b.out_rows, b.out_cols)


def run_gpu(b, runs=1):
    """-> (output [out_rows, out_cols], the per-op run_profiled records).  The Engine is closed before returning.

    The output is NaN-poisoned before every run, as Sim poisons its own: consecutive cases often have the same shape
    and the same reference, and the caching allocator hands a case the block the previous case's result was just
    copied out of -- an output element a kernel never stores must show, not pass on the previous engine's answer."""
    import torch
    from mvector.engine import Engine, Program
    eng = Engine()
    try:
        eng.load_weights(b.blob)
        prog = Program(eng, b.pb)
        y = torch.empty(b.out_rows, b.out_cols, device='cuda')
        x = torch.from_numpy(b.X).cuda().contiguous()
        for _ in range(runs):
            y.fill_(float('nan'))
            ops = prog.run_profiled(x, y)
        torch.cuda.synchronize()
        return y.cpu().numpy(), ops
    finally:
        eng.close()


def program_engines(prog):
    """Resolved engine of every op of a Program (vp_program_op_info), without running it."""
    import ctypes as C
    out = []
    for i in range(prog.n_ops):
        kind, eng = C.c_int32(), C.c_int32()
        M, N, K = C.c_int64(), C.c_int64(), C.c_int64()
        L.lib().vp_program_op_info(prog._p, i, C.byref(kind), C.byref(M), C.byref(N), C.byref(K), C.byref(eng))
        out.append(eng.value)
    return out


def assert_engines(b, ops):
    """Every conv op ran on the engine its case requested (no silent TC16 -> TF32 or TC -> FFMA fallback)."""
    for i, want in b.expect.items():
        if b.pb.ops[i].kind == L.OP_CONV:
            assert ops[i]['engine'] == want, (i, ops[i], want)


# ---------------------------------------------------------------------------------------------------------------
# mirrors of the launchers' kernel choices (coverage-intent checks, tests/test_op_edges_cpu.py)
# ---------------------------------------------------------------------------------------------------------------
def tc_schedule(o, engine):
    """Tile / chunk schedule of a tensor-core conv: conv_tc.cu launch_conv_tc_impl (:593-597, :609-611)."""
    K = o.KT * o.KF * (o.Cin + (o.Cin2 if o.src2_mode == L.SRC2_CONCAT else 0))
    M = o.B * o.Tout * o.Fout
    bke = 64 if engine == L.ENGINE_TC16 else 32                     # :588
    bn = tc_tile_n(o.Cout, o.tc_kc > 0)                             # :563-566 (mirrored by engine.tc_tile_n)
    m_tiles, n_tiles = (M + 127) // 128, (o.Cout + bn - 1) // bn     # :593-594
    k_blocks = (K + bke - 1) // bke                                 # :595
    kc = o.tc_kc // bke if 0 < o.tc_kc < K else k_blocks            # :596
    n_chunks = (k_blocks + kc - 1) // kc                            # :597
    tiles = m_tiles * n_tiles
    grid = min(SMS, tiles)                                          # :609-611
    # :372-376: the epilogue is `simple` without ubias / gate / sum and with act, act2 in {none, ReLU, Hardtanh(0, 20)};
    # :438: a tile takes the fast epilogue when it is simple and has no row / column tail
    clamps = (L.ACT_NONE, L.ACT_RELU, L.ACT_HARDTANH20)
    simple = (o.ubias == L.BUF_NONE and o.gate == L.BUF_NONE and o.sum == L.BUF_NONE and o.act in clamps
              and o.act2 in clamps)
    tiles_per_cta = -(-tiles // grid)                               # :194 my_tiles of CTA 0, the busiest
    return dict(bn=bn, m_tiles=m_tiles, n_tiles=n_tiles, tiles=tiles, tiles_per_cta=tiles_per_cta,
                k_blocks=k_blocks, kc=kc, n_chunks=n_chunks, last_chunk=k_blocks - (n_chunks - 1) * kc,
                items=tiles_per_cta * k_blocks,                     # :195 total_items: the producers' (tile, K block) stream
                k_tail=K % 32, m_tail=M % 128, simple=simple,
                fast=simple and M % 128 == 0 and o.Cout % bn == 0)     # every tile on the fast epilogue


def small_m_ok(o):
    """conv_ffma.cu:219-222 (small_m_ok)."""
    K = o.KT * o.KF * (o.Cin + (o.Cin2 if o.src2_mode == L.SRC2_CONCAT else 0))
    return (o.B * o.Tout * o.Fout <= 1024 and o.KT == 1 and o.KF == 1 and o.sT == 1 and o.sF == 1 and o.padT == 0
            and o.padF == 0 and o.src2_mode == L.SRC2_NONE and o.pre_s < 0 and o.Tin == o.Tout and o.Fin == o.Fout
            and K % 4 == 0)


def c1_wide(o):
    """conv_ffma.cu:366-367 (launch_conv_c1: the wide variant's predicate)."""
    return (o.ubias == L.BUF_NONE and o.gate == L.BUF_NONE and o.res == L.BUF_NONE and o.sum == L.BUF_NONE
            and o.Cout in (16, 32, 64) and o.KT * o.KF <= 49 and o.out_ld % 4 == 0 and o.out_coff % 4 == 0)


def tc_supported(o):
    """conv_tc.cu:568-578 (conv_tc_supported) on a lowered op; fill_conv (api.cu:628-648) gives M, N, K and w_tc."""
    K = o.KT * o.KF * (o.Cin + (o.Cin2 if o.src2_mode == L.SRC2_CONCAT else 0))
    return (o.w_tc >= 0 and o.B * o.Tout * o.Fout >= 1024 and o.Cout >= 16 and o.Cout % 4 == 0 and K % 4 == 0
            and o.tc_kc >= 0 and o.tc_kc % 64 == 0 and o.tc_bn == tc_tile_n(o.Cout, o.tc_kc > 0)
            and not (o.pre_s >= 0 and o.src2_mode != L.SRC2_NONE))


def tc16_supported(o):
    """conv_tc.cu:635-641 (conv_tc16_supported): MODE 0 only, a tracked source (amax slot, PlanBuilder.finalize), Cin,
    CinTot and K multiples of 8, N >= 128."""
    cin_tot = o.Cin + (o.Cin2 if o.src2_mode == L.SRC2_CONCAT else 0)
    return (tc_supported(o) and o.amax_in > 0 and o.pre_s < 0 and o.src2_mode != L.SRC2_ADD and o.Cin % 8 == 0
            and cin_tot % 8 == 0 and o.KT * o.KF * cin_tot % 8 == 0 and o.Cout >= 128)


TC16_ON = not os.environ.get('VPB_TC_F16', '').startswith('0')      # api.cu:79-83 (tc16_enabled)


def engine_of(o, pref=None, tc16_on=None):
    """Engine vp_program_create resolves for a lowered, finalized op (api.cu:559-583): ``pref`` is the requested engine
    (default: the op's own), ``tc16_on`` whether AUTO may pick the fp16 split (default: VPB_TC_F16 as the library reads
    it).  0 for ops that are not CONV; ValueError where the library refuses the program (VP_ERR_UNSUPPORTED)."""
    if o.kind != L.OP_CONV:
        return 0
    pref = o.engine if pref is None else pref
    tc16_on = TC16_ON if tc16_on is None else tc16_on
    ok = tc_supported(o)
    ok16 = ok and o.w_tc16_q > 0 and o.tc16_descale > 0 and tc16_supported(o)
    if (pref == L.ENGINE_TC and not ok) or (pref == L.ENGINE_TC16 and not ok16):
        raise ValueError('shape / operands not supported by the requested tensor-core engine')
    if pref == L.ENGINE_TC16 or (pref == L.ENGINE_AUTO and ok16 and tc16_on):
        return L.ENGINE_TC16
    if pref == L.ENGINE_TC or (pref == L.ENGINE_AUTO and ok):
        return L.ENGINE_TC
    return L.ENGINE_FFMA


def _tc_suffix(pre, add):
    """conv_tc.cu:621-624: the prologue selects conv_tc_kernel<2, ...>, else an added second source <1, ...>, else <0>."""
    return ',pre' if pre else ',add' if add else ''


def kernel_of(o, engine):
    """Name of the kernel a lowered op launches with the given resolved conv engine."""
    if o.kind == L.OP_CONV_C1:
        return 'conv_c1_wide' if c1_wide(o) else 'conv_c1'
    if o.kind == L.OP_CONV:
        if engine == L.ENGINE_TC16:
            return 'conv_tc<f16>'
        if engine == L.ENGINE_TC:
            return 'conv_tc<tf32%s>' % _tc_suffix(o.pre_s >= 0, o.src2_mode == L.SRC2_ADD)
        if small_m_ok(o):
            return 'linear_small_m'
        # conv_ffma.cu:231-240: BN = 128 above N = 64, 64 above N = 32, else 32
        return 'conv_ffma<%d>' % (128 if o.Cout > 64 else 64 if o.Cout > 32 else 32)
    if o.kind == L.OP_POOL2D:
        return 'pool2d'
    if o.kind == L.OP_EW:
        return 'pad_copy' if o.mode == L.EW_PAD_COPY else 'ew'
    if o.kind == L.OP_COLSTATS:
        R = o.Tin * o.Fin
        # pool.cu:157: staged strip for the non-segment modes up to 100 KB on 4-float aligned views
        staged = (o.mode != L.STATS_SEG_CONTEXT and R * 128 <= 100 * 1024 and o.Cin % 4 == 0 and o.in_ld % 4 == 0
                  and o.in_coff % 4 == 0)
        return 'colstats_smem' if staged else 'colstats'
    if o.kind == L.OP_ASP_POOL:
        # pool.cu:256: both [T, 32] strips staged up to 200 KB on 4-float aligned views
        staged = (o.Tin * 256 <= 200 * 1024 and o.Cin % 4 == 0 and o.in_ld % 4 == 0 and o.in_coff % 4 == 0
                  and o.src2_ld % 4 == 0 and o.src2_coff % 4 == 0)
        return 'asp_smem' if staged else 'asp'
    raise ValueError(o.kind)


BENCH_T = dict(c2=298, c3=298, c4=251, c5=998)     # frames: 3 s Fbank (25 / 10 ms), 5 s Mel (hop 320, centred), 10 s


def bench_model(name):
    """The bench.py configuration's backbone mirror with its seeded weights (oracle.models.random_state_dict, as
    bench.save_weights); lowering it needs no GPU."""
    import bench
    from oracle import models as om
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object
    cfg = bench.CONFIGS[name]
    gain = getattr(om, 'CONDITIONED_GAIN', {}).get(cfg['model'])
    sd = om.random_state_dict(cfg['model'], cfg['fdim'], seed=0, **(dict(gain=gain) if gain is not None else {}),
                              **cfg['margs'])
    model = build_model(cfg['fdim'], dict_to_object({'model_conf': {'model': cfg['model'], 'model_args': cfg['margs']}}))
    model.load_state_dict(sd)
    return model, cfg


def ew_grid_strides(o):
    """True when the ew / pool2d grid (capped at 132 * 32 CTAs of 256 threads, pool.cu:330-332 / :377-380) is smaller
    than the float4 count, i.e. the grid-stride loop runs more than once."""
    rows = o.B * (o.Tout * o.Fout if o.kind == L.OP_POOL2D else o.Tin * o.Fin)
    return rows * (o.Cin // 4) > 132 * 32 * 256


# ---------------------------------------------------------------------------------------------------------------
# case tables
# ---------------------------------------------------------------------------------------------------------------
def _tc(name, engines, table=None, **c):
    """A tensor-core conv case, once per engine ('tc' = split TF32, 'tc16' = fp16 split, 'ffma' = exact reference),
    into ``table`` (TC_CASES by default)."""
    for e in engines:
        kern = {'tc': 'conv_tc<tf32%s>' % _tc_suffix(c.get('pre'), c.get('src2_mode') == L.SRC2_ADD),
                'tc16': 'conv_tc<f16>',
                'ffma': 'conv_ffma<%d>' % (128 if c['N'] > 64 else 64 if c['N'] > 32 else 32)}[e]
        (TC_CASES if table is None else table)[f'{name}-{e}'] = dict(c, op='conv', engine=e, kernel=kern)


TC_CASES = {}
# persistent schedule: several tiles per CTA (cross-tile gather cursor, stage / phase carry-over, next-tile residual
# prefetch, a chunked layer running tile after tile); 16 x 1000 rows, N = 512, K = 2048 chunked by 512 -> 125 x 8 tiles
_tc('multi_tile_1000', ('tc', 'tc16'), seed=101, B=16, Tin=1000, Cin=2048, N=512, bias=True, res=True, ubias=True,
    act=L.ACT_RELU, intent=dict(tiles=1000, tiles_per_cta=8, n_chunks=4))
# 133 tiles on 132 CTAs: exactly one CTA runs a second tile (7 x 2420 rows, N = 128)
_tc('tiles_133', ('tc', 'tc16'), seed=102, B=7, Tin=2420, Cin=64, N=128, bias=True, act=L.ACT_RELU, post=True,
    res=True, intent=dict(tiles=133, tiles_per_cta=2))
# M = 2049 (M % 128 == 1) and every N-tile composition: BN = 32 (n32), 48 (n32+n16), 64, 80 (n64+n16), 96 (n64+n32),
# 112 (n64+n32+n16), 128 and two 128-wide tiles with 4 / 68 columns in the second
for _i, _N in enumerate((20, 36, 52, 68, 84, 100, 116, 132, 196)):
    _tc(f'm_tail1_n{_N}', ('tc', 'tc16') if _N >= 128 else ('tc',), seed=110 + _i, B=3, Tin=683, Cin=64, N=_N,
        bias=True, act=L.ACT_RELU, post=True, intent=dict(m_tail=1))
# M = 2048: every tile is full, so every tile takes the fast epilogue (bias / ReLU / affine / residual)
_tc('m_full_fast', ('tc', 'tc16'), seed=120, B=4, Tin=512, Cin=96, N=256, bias=True, act=L.ACT_RELU, post=True,
    res=True, act2=L.ACT_RELU, intent=dict(fast=True))
# K edges: K < 32, K not a multiple of 32 / 64, CinTot < 32 (one K block spans several taps)
_tc('k4_1x1', ('tc',), seed=130, B=3, Tin=683, Cin=4, N=64, bias=True)
_tc('k12_k3_cin4', ('tc',), seed=131, B=3, Tin=683, Cin=4, N=64, KT=3, padT=1, bias=True, act=L.ACT_RELU)
_tc('k20_k5_cin4', ('tc',), seed=132, B=3, Tin=683, Cin=4, N=48, KT=5, padT=2, bias=True)
_tc('k72_1x1', ('tc', 'tc16'), seed=133, B=3, Tin=683, Cin=72, N=128, bias=True)
_tc('k120_k3_cin40', ('tc', 'tc16'), seed=134, B=3, Tin=683, Cin=40, N=128, KT=3, padT=1, bias=True, act=L.ACT_RELU)
_tc('k72_3x3_cin8', ('tc', 'tc16'), seed=135, B=2, Tin=40, Fin=20, Cin=8, N=128, KT=3, KF=3, padT=1, padF=1,
    bias=True, act=L.ACT_HARDTANH20)
# accumulation-chunk remainders: ERes2Net's (512, 256) policy at K = 576 / 1152 / 2304, the default at K = 1600
_tc('eres_k576', ('tc', 'tc16'), seed=140, policy=ERES_POLICY, B=2, Tin=40, Fin=20, Cin=64, N=128, KT=3, KF=3,
    padT=1, padF=1, bias=True, act=L.ACT_HARDTANH20, res=True, intent=dict(chunk_remainder=True))
_tc('eres_k1152', ('tc', 'tc16'), seed=141, policy=ERES_POLICY, B=2, Tin=40, Fin=20, Cin=128, N=128, KT=3, KF=3,
    padT=1, padF=1, bias=True, act=L.ACT_RELU, intent=dict(chunk_remainder=True))
_tc('eres_k2304', ('tc', 'tc16'), seed=142, policy=ERES_POLICY, B=2, Tin=20, Fin=40, Cin=256, N=128, KT=3, KF=3,
    padT=1, padF=1, bias=True, post=True, intent=dict(n_chunks=9))
_tc('default_k1600', ('tc', 'tc16'), seed=143, B=4, Tin=300, Cin=320, N=128, KT=5, padT=2, bias=True, act=L.ACT_RELU,
    intent=dict(chunk_remainder=True))
# reflect padding at the smallest Tin the validator accepts (Tin = dilation + 1)
for _d in (2, 3):
    _tc(f'reflect_min_tin_d{_d}', ('ffma', 'tc', 'tc16'), seed=150 + _d, B=1200 // (_d + 1), Tin=_d + 1, Cin=64,
        N=128, KT=3, dT=_d, padT=_d, pad_mode=L.PAD_REFLECT, bias=True, act=L.ACT_RELU)
# fp16-split epilogues (general path): per-segment gate, residual, accumulate-into, SiLU / sigmoid / tanh, and a
# channel concat whose two halves are windows of one allocation
_tc('gate_seg', ('tc', 'tc16'), seed=160, B=6, Tin=249, Cin=128, N=128, KT=3, dT=2, padT=2, gate=True, seg_len=100,
    n_seg=3)
_tc('res_tail', ('tc', 'tc16'), seed=161, B=4, Tin=300, Cin=128, N=192, bias=True, act=L.ACT_RELU, res=True)
_tc('sum_into', ('tc', 'tc16'), seed=162, B=4, Tin=300, Cin=64, N=128, bias=True, act=L.ACT_RELU, post=True, sum=True)
_tc('silu', ('tc', 'tc16'), seed=163, B=4, Tin=300, Cin=64, N=128, bias=True, act=L.ACT_SILU, ubias=True)
_tc('sigmoid_act2', ('tc', 'tc16'), seed=164, B=4, Tin=300, Cin=64, N=128, bias=True, post=True, act2=L.ACT_SIGMOID)
_tc('tanh_act2_res', ('tc', 'tc16'), seed=165, B=4, Tin=300, Cin=64, N=128, bias=True, res=True, act2=L.ACT_TANH)
_tc('concat_one_alloc', ('tc', 'tc16'), seed=166, B=4, Tin=300, Cin=64, Cin2=64, src2_mode=L.SRC2_CONCAT, N=128,
    bias=True, act=L.ACT_SILU, in_coff=8)
# output column window inside a wider matrix (Res2 concat buffers)
_tc('out_window', ('ffma', 'tc'), seed=167, B=4, Tin=300, Cin=64, N=64, bias=True, act=L.ACT_RELU, out_coff=32,
    in_coff=4)

# ---- the add (conv_tc_kernel<1, ...>) and BN-ReLU prologue (conv_tc_kernel<2, ...>) gathers ----
# Both run a 2-deep register pipeline (conv_tc.cu:275, refill :339, publish loop :350-354) with their own slots (:131-132)
# and publish arithmetic (:322-329).  Every case also runs on the FFMA engine, whose gather_a4 (common.cuh:159-190)
# computes the same operand, and has a MODE 0 twin (tests/test_gpu_conv_gathers.py).  Prologue scales are signed powers
# of two (the twin needs x * s exact).
ADD, PRE = dict(src2_mode=L.SRC2_ADD), dict(pre='pow2')
_GE = ('tc', 'ffma')
# M = 2049 (a one-row M tail) and every N tile: BN = 16, then 32 ... 128 with a 12-column tail in the last tile.  The
# ECAPA Res2 add (K = 192, dilation 2, reflect / zero padding alternating); the CAM++ prologue on a column window of a
# wider map (in_ld > Cin, in_coff = 8), 1x1 and KT = 3 with zero padding alternating
for _i, _N in enumerate((16, 20, 36, 52, 68, 84, 100, 116)):
    _bn = max(16, (_N + 15) // 16 * 16)
    _tc(f'add_m_tail1_n{_N}', _GE, **ADD, seed=500 + _i, B=3, Tin=683, Cin=64, N=_N, KT=3, dT=2, padT=2,
        pad_mode=L.PAD_REFLECT if _i % 2 == 0 else L.PAD_ZERO, bias=True, act=L.ACT_RELU, post=True,
        intent=dict(m_tail=1, bn=_bn))
    _tc(f'pre_m_tail1_n{_N}', _GE, **PRE, seed=520 + _i, B=3, Tin=683, Cin=64, in_coff=8, N=_N,
        **(dict(KT=3, padT=1) if _i % 2 else {}), bias=True, act=L.ACT_RELU, post=True, intent=dict(m_tail=1, bn=_bn))
# accumulation-chunk remainders: the add under ERes2Net's (512, 256) policy on a zero-padded 3x3 map with odd Fin
# (K = 576: 18 K blocks in chunks of 8, 8, 2); the prologue under the default policy (K = 1600: 16, 16, 16, 2)
_tc('add_eres_k576_3x3_odd_fin', _GE, **ADD, seed=540, policy=ERES_POLICY, B=2, Tin=40, Fin=21, Cin=64, N=64, KT=3,
    KF=3, padT=1, padF=1, bias=True, act=L.ACT_HARDTANH20, res=True, intent=dict(chunk_remainder=True))
_tc('pre_default_k1600', _GE, **PRE, seed=541, B=4, Tin=300, Cin=320, N=128, KT=5, padT=2, bias=True, act=L.ACT_RELU,
    intent=dict(chunk_remainder=True))
# 133 tiles on 132 CTAs: exactly one CTA runs a second tile
_tc('add_tiles_133', _GE, **ADD, seed=542, B=7, Tin=2420, Cin=64, N=128, KT=3, dT=3, padT=3, pad_mode=L.PAD_REFLECT,
    bias=True, act=L.ACT_RELU, post=True, intent=dict(tiles=133, tiles_per_cta=2))
_tc('pre_tiles_133', _GE, **PRE, seed=543, B=7, Tin=2420, Cin=128, N=128, bias=True, act=L.ACT_RELU, post=True, res=True,
    intent=dict(tiles=133, tiles_per_cta=2))
# 64 x 1056 rows = 528 full tiles, 4 per CTA, every one on the fast epilogue; K = 108 (4 K blocks, a K tail of 12)
_tc('add_4_tiles_per_cta_k_tail', _GE, **ADD, seed=544, B=64, Tin=1056, Cin=36, N=64, KT=3, dT=4, padT=4,
    pad_mode=L.PAD_REFLECT, bias=True, act=L.ACT_RELU, post=True, res=True,
    intent=dict(tiles_per_cta=4, k_tail=12, fast=True))
_tc('pre_4_tiles_per_cta_k_tail', _GE, **PRE, seed=545, B=64, Tin=1056, Cin=36, N=128, KT=3, padT=1, bias=True,
    act=L.ACT_RELU, post=True, act2=L.ACT_RELU, intent=dict(tiles_per_cta=4, k_tail=12, fast=True))
# one K block per tile and 3 tiles per CTA (48 x 1056 rows = 396 tiles): the 2-deep pipeline refills across tiles on
# every item and ends on an odd item; the general epilogue through a feature (ubias + SiLU, gate + tanh)
_tc('add_kb1_odd_items_ubias_silu', _GE, **ADD, seed=546, B=48, Tin=1056, Cin=32, N=48, bias=True, ubias=True,
    act=L.ACT_SILU, intent=dict(k_blocks=1, tiles_per_cta=3, items=3, simple=False))
_tc('pre_kb1_odd_items_gate_tanh', _GE, **PRE, seed=547, B=48, Tin=1056, Cin=8, N=32, KT=3, padT=1, bias=True,
    gate=True, act2=L.ACT_TANH, intent=dict(k_blocks=1, k_tail=24, tiles_per_cta=3, items=3, simple=False))
# add: reflect padding at the smallest map the validator accepts (Tin = dilation + 1), dilations 2, 3, 4 of ECAPA's Res2
for _d in (2, 3, 4):
    _tc(f'add_reflect_min_tin_d{_d}', _GE, **ADD, seed=548 + _d, B=1200 // (_d + 1), Tin=_d + 1, Cin=64, N=64, KT=3,
        dT=_d, padT=_d, pad_mode=L.PAD_REFLECT, bias=True, act=L.ACT_RELU, post=True)
# add: the second source in an allocation of its own, row pitch 84 and first column 12 (x: the program input, pitch =
# its width, first column 4), accumulated into a view (general epilogue)
_tc('add_src2_own_alloc', _GE, **ADD, seed=553, B=4, Tin=300, Cin=64, N=128, KT=3, padT=1, in_coff=4, src2_width=84,
    src2_coff=12, bias=True, act=L.ACT_RELU, sum=True)
# prologue: zero padding on a 3x3 map (okmask keeps padded taps at 0, not at relu(h)), reflect padding, no ReLU, and
# CAM++'s last transit (N = 512, K = 1024, BN affine + ReLU after the conv)
_tc('pre_3x3_zero_pad', _GE, **PRE, seed=554, B=2, Tin=40, Fin=21, Cin=32, N=32, KT=3, KF=3, padT=1, padF=1, bias=True,
    act=L.ACT_RELU)
_tc('pre_reflect_d2', _GE, **PRE, seed=555, B=4, Tin=300, Cin=64, N=64, KT=3, dT=2, padT=2, pad_mode=L.PAD_REFLECT,
    bias=True, act=L.ACT_RELU, post=True)
_tc('pre_no_relu_zero_pad', _GE, **PRE, pre_relu=False, seed=556, B=4, Tin=300, Cin=64, N=96, KT=3, padT=1,
    bias=True, post=True)
_tc('pre_cam_transit_n512_k1024', _GE, **PRE, seed=557, B=4, Tin=300, Cin=1024, N=512, post=True, act2=L.ACT_RELU)
GATHER_CASES = {n: c for n, c in TC_CASES.items() if c.get('pre') or c.get('src2_mode') == L.SRC2_ADD}

# position invariance: the rows of the first three utterances must not depend on the batch around them.  At B = 16 the
# 16000 rows are 125 full tiles (fast epilogue, ~8 tiles per CTA); at B = 3 the last tile is a tail (general path).
# Variants: the plain source, the added second source, the prologue.
INVARIANCE = dict(op='conv', seed=170, B=16, Tin=1000, Cin=2048, N=512, bias=True, act=L.ACT_RELU, post=True, res=True)
INVARIANCE_VARIANTS = {'': {}, 'add': ADD, 'pre': PRE}


def invariance(variant, engine, B):
    return dict(INVARIANCE, **INVARIANCE_VARIANTS[variant], engine=engine, B=B)


# ---- the backbones' conv geometries on both engines, and on the fp16 split where N >= 128 and nothing but a plain
# source feeds it: pointwise GEMMs, Res2 k3 convs with dilation, reflect padding and an added or accumulated second
# source, stems, valid TDNN convs, 2-D 3x3 convs with stride / residual / concat, CAM++'s BN-ReLU prologue (uniform
# scales) and per-segment gate, K chunked by the default policy, N and K tails ----
ENGINE_CASES = {}
_TC16_GEOMETRIES = {'gemm_512', 'gemm_n1536_k128', 'gemm_k1536_n128_ubias_tanh', 'stem_k5_reflect', 'tdnn_valid_k3_d3',
                    'k5_stride2_zero', 'n_tail_192', 'long_k_chunked_9216', 'long_k_chunked_4096_n128'}
for _name, _c in dict(
        gemm_512=dict(seed=1, B=8, Tin=298, Cin=512, N=512, bias=True, act=L.ACT_RELU, post=True),
        gemm_n1536_k128=dict(seed=2, B=5, Tin=298, Cin=128, N=1536, bias=True),
        gemm_k1536_n128_ubias_tanh=dict(seed=3, B=6, Tin=211, Cin=1536, N=128, ubias=True, act=L.ACT_RELU, post=True,
                                        act2=L.ACT_TANH),
        res2_k3_dil2_reflect_add=dict(seed=4, B=9, Tin=298, Cin=64, N=64, KT=3, dT=2, padT=2, pad_mode=L.PAD_REFLECT,
                                      bias=True, act=L.ACT_RELU, post=True, src2_mode=L.SRC2_ADD),
        stem_k5_reflect=dict(seed=5, B=7, Tin=298, Cin=80, N=512, KT=5, padT=2, pad_mode=L.PAD_REFLECT, bias=True,
                             act=L.ACT_RELU, post=True),
        tdnn_valid_k3_d3=dict(seed=6, B=4, Tin=300, Tout=294, Cin=512, N=512, KT=3, dT=3, bias=True, act=L.ACT_RELU,
                              post=True),
        conv2d_3x3_s2=dict(seed=7, B=3, Tin=61, Fin=40, Tout=31, Fout=20, Cin=32, N=48, KT=3, KF=3, sT=2, sF=2, padT=1,
                           padF=1, bias=True, act=L.ACT_HARDTANH20),
        conv2d_3x3_res_relu=dict(seed=8, B=2, Tin=50, Fin=20, Cin=32, N=32, KT=3, KF=3, padT=1, padF=1, bias=True,
                                 res=True, act2=L.ACT_RELU),
        concat_1x1_silu=dict(seed=9, B=2, Tin=40, Fin=30, Cin=16, Cin2=16, N=16, bias=True, act=L.ACT_SILU,
                             src2_mode=L.SRC2_CONCAT),
        cam_pre_bn_relu=dict(seed=10, B=9, Tin=149, Cin=160, N=128, pre=True, bias=True, act=L.ACT_RELU),
        cam_local_gate_seg=dict(seed=11, B=6, Tin=249, Cin=128, N=32, KT=3, dT=2, padT=2, gate=True, seg_len=100,
                                n_seg=3),
        k5_stride2_zero=dict(seed=12, B=8, Tin=298, Tout=149, Cin=320, N=128, KT=5, sT=2, padT=2, bias=True,
                             act=L.ACT_RELU),
        n_tail_192=dict(seed=13, B=3, Tin=400, Cin=96, N=192, bias=True),
        long_k_chunked_9216=dict(seed=15, B=6, Tin=40, Fin=20, Tout=20, Fout=10, Cin=1024, N=256, KT=3, KF=3, sT=2,
                                 sF=2, padT=1, padF=1),
        long_k_chunked_4096_n128=dict(seed=16, B=7, Tin=151, Cin=4096, N=128, ubias=True, act=L.ACT_RELU, post=True,
                                      act2=L.ACT_TANH),
        res2_k3_dil3_reflect_sum=dict(seed=17, B=9, Tin=298, Cin=64, N=64, KT=3, dT=3, padT=3, pad_mode=L.PAD_REFLECT,
                                      bias=True, act=L.ACT_RELU, post=True, sum=True),
        conv2d_3x3_sum_hardtanh=dict(seed=18, B=2, Tin=50, Fin=20, Cin=16, N=16, KT=3, KF=3, padT=1, padF=1, bias=True,
                                     act=L.ACT_HARDTANH20, sum=True),
        k_tail_72=dict(seed=14, B=11, Tin=100, Cin=24, N=24, KT=3, padT=1, bias=True, act=L.ACT_HARDTANH20),
).items():
    _tc(_name, ('ffma', 'tc', 'tc16') if _name in _TC16_GEOMETRIES else ('ffma', 'tc'), table=ENGINE_CASES, **_c)

# ---- engine routing: what AUTO resolves to where a tensor-core engine cannot take the op, and the explicit requests
# vp_program_create refuses (VP_ERR_UNSUPPORTED; engine_of raises ValueError) rather than run differently ----
REFUSED_CASES = {}
# a BN-ReLU prologue combined with a second source: the tensor-core gather reads one source, so AUTO runs FFMA
for _name, _c in dict(
        pre_concat_1x1=dict(seed=21, B=9, Tin=149, Cin=96, Cin2=64, N=128, pre=True, bias=True, act=L.ACT_RELU,
                            src2_mode=L.SRC2_CONCAT),
        pre_add_k3=dict(seed=22, B=9, Tin=149, Cin=64, N=64, KT=3, padT=1, pre=True, bias=True, act=L.ACT_RELU,
                        src2_mode=L.SRC2_ADD),
).items():
    _tc(_name, ('ffma',), table=ENGINE_CASES, **_c)
    ENGINE_CASES[f'{_name}-auto'] = dict(ENGINE_CASES[f'{_name}-ffma'], engine='auto')
    REFUSED_CASES[f'{_name}-tc'] = dict(_c, op='conv', engine='tc')
# a conv reading the program input itself has no amax slot: AUTO runs split TF32
_RAW = dict(op='conv', seed=23, B=8, Tin=200, Cin=256, N=256, raw_input=True)
ENGINE_CASES['raw_input-auto'] = dict(_RAW, engine='auto', kernel='conv_tc<tf32>')
REFUSED_CASES['raw_input-tc16'] = dict(_RAW, engine='tc16')

FFMA_CASES = {}
# linear_small_m_kernel: M <= 1024 pointwise linears (SE MLPs, ASP per-utterance bias, final FC)
for _name, _c in dict(
        m1_k4_n4=dict(B=1, Tin=1, Cin=4, N=4, bias=True),
        m1_k3072_n28_tanh=dict(B=1, Tin=1, Cin=3072, N=28, post=True, act2=L.ACT_TANH),
        m7_k124_n28_ubias_tanh=dict(B=7, Tin=1, Cin=124, N=28, ubias=True, act=L.ACT_TANH),
        m7_k128_n4_sigmoid=dict(B=7, Tin=1, Cin=128, N=4, bias=True, act=L.ACT_SIGMOID),
        m8_k128_n36_gate_sigmoid=dict(B=8, Tin=1, Cin=128, N=36, gate=True, act2=L.ACT_SIGMOID, bias=True),
        m8_k132_n192_res=dict(B=8, Tin=1, Cin=132, N=192, bias=True, res=True, act2=L.ACT_RELU),
        m9_k132_n192_res=dict(B=3, Tin=3, Cin=132, N=192, bias=True, res=True, act2=L.ACT_RELU),
        m9_k4_n36_sum=dict(B=3, Tin=3, Cin=4, N=36, bias=True, sum=True),
        m1023_k3072_n192_ubias=dict(B=3, Tin=341, Cin=3072, N=192, ubias=True, act=L.ACT_RELU, post=True),
        m1023_k124_n4_gate=dict(B=3, Tin=341, Cin=124, N=4, gate=True, act=L.ACT_TANH),
        m1024_k132_n36_sum=dict(B=4, Tin=256, Cin=132, N=36, bias=True, sum=True),
        m1024_k3072_n28_gate=dict(B=4, Tin=256, Cin=3072, N=28, gate=True, act2=L.ACT_SIGMOID),
        m1024_k128_n192_window=dict(B=4, Tin=256, Cin=128, N=192, bias=True, in_coff=4, out_coff=12),
).items():
    FFMA_CASES[f'small_m_{_name}'] = dict(_c, op='conv', engine='ffma', kernel='linear_small_m', seed=200 + len(FFMA_CASES))
# one row above the small-M limit: the tiled kernel
FFMA_CASES['tiled_m1025'] = dict(op='conv', engine='ffma', kernel='conv_ffma<64>', seed=230, B=5, Tin=205, Cin=128,
                                 N=36, bias=True, ubias=True, act=L.ACT_TANH)
# conv_ffma_kernel<32|64|128> with M = 2049 (one row in the last M tile), K = 60 (a K tail of 12 in the 16-wide K loop)
for _N, _bn in ((4, 32), (36, 64), (68, 128), (132, 128)):
    FFMA_CASES[f'tiled_m2049_n{_N}'] = dict(op='conv', engine='ffma', kernel=f'conv_ffma<{_bn}>', seed=240 + _N, B=3,
                                            Tin=683, Cin=20, N=_N, KT=3, padT=1, bias=True, act=L.ACT_RELU,
                                            res=_N == 68, gate=_N == 132)
# 2-D stems (CONV_C1): the wide kernel (N = 16 / 32 / 64, plain epilogue) and the generic one
C1_CASES = dict(
    wide_n16_3x3=dict(kernel='conv_c1_wide', B=3, Tin=61, Fin=40, N=16, KT=3, KF=3, padT=1, padF=1, bias=True,
                      act=L.ACT_RELU, post=True),
    wide_n32_3x3_odd_m=dict(kernel='conv_c1_wide', B=1, Tin=37, Fin=41, N=32, KT=3, KF=3, padT=1, padF=1, bias=True,
                            act=L.ACT_RELU),
    wide_n64_7x7_s3_odd_m=dict(kernel='conv_c1_wide', B=3, Tin=101, Fin=83, Tout=33, Fout=27, N=64, KT=7, KF=7, sT=3,
                               sF=3, padT=1, padF=1, bias=True, act=L.ACT_RELU),
    wide_n32_window=dict(kernel='conv_c1_wide', B=2, Tin=30, Fin=21, N=32, KT=3, KF=3, padT=1, padF=1, bias=True,
                         act2=L.ACT_HARDTANH20, out_coff=8),
    generic_n8=dict(kernel='conv_c1', B=2, Tin=31, Fin=40, N=8, KT=3, KF=3, padT=1, padF=1, bias=True, act=L.ACT_RELU),
    generic_n48_7x7_s3=dict(kernel='conv_c1', B=2, Tin=100, Fin=80, Tout=32, Fout=26, N=48, KT=7, KF=7, sT=3, sF=3,
                            padT=1, padF=1, bias=True, act=L.ACT_RELU, post=True),
    generic_n32_res=dict(kernel='conv_c1', B=2, Tin=31, Fin=40, N=32, KT=3, KF=3, padT=1, padF=1, bias=True,
                         res=True, act2=L.ACT_RELU),
    generic_n32_gate=dict(kernel='conv_c1', B=3, Tin=31, Fin=40, N=32, KT=3, KF=3, padT=1, padF=1, bias=True,
                          gate=True, act=L.ACT_SIGMOID),
)
for _i, (_name, _c) in enumerate(C1_CASES.items()):
    FFMA_CASES[f'c1_{_name}'] = dict(_c, op='c1', Cin=1, seed=260 + _i)

_P, _E = dict(op='pool2d', kernel='pool2d'), dict(op='ew', kernel='ew')
GLUE_CASES = dict(
    pool_max_k3s1=dict(_P, mode='max', B=2, Tin=31, Fin=21, C=16, stride=1),
    pool_max_k3s2_negative=dict(_P, mode='max', B=2, Tin=31, Fin=21, C=32, stride=2, fill='negative'),
    pool_max_fout1_negative=dict(_P, mode='max', B=3, Tin=9, Fin=1, C=16, stride=2, fill='negative'),
    pool_avg_k3s1=dict(_P, mode='avg', B=2, Tin=31, Fin=21, C=16, stride=1),
    pool_avg_k3s2_fout1=dict(_P, mode='avg', B=3, Tin=9, Fin=2, C=16, stride=2),
    pool_avg_s2_window=dict(_P, mode='avg', B=2, Tin=33, Fin=19, C=24, stride=2, in_coff=8, out_coff=48),
    ew_gate=dict(_E, mode='GATE_RES', B=3, T=97, C=36, gate=True),
    ew_gate_relu=dict(_E, mode='GATE_RES', B=3, T=97, C=36, gate=True, act2=L.ACT_RELU),
    ew_res=dict(_E, mode='GATE_RES', B=3, T=97, C=36, res=True),
    ew_res_relu=dict(_E, mode='GATE_RES', B=3, T=97, C=36, res=True, act2=L.ACT_RELU),
    ew_gate_res=dict(_E, mode='GATE_RES', B=3, T=97, C=36, gate=True, res=True),
    ew_gate_res_relu=dict(_E, mode='GATE_RES', B=3, T=97, C=36, gate=True, res=True, act2=L.ACT_RELU),
    ew_gate_res_window=dict(_E, mode='GATE_RES', B=3, T=97, C=36, gate=True, res=True, in_coff=4, out_coff=20),
    ew_aff_saturated=dict(_E, mode='AFF', B=3, T=97, C=64, saturate=True),
    ew_aff_window=dict(_E, mode='AFF', B=3, T=97, C=64, in_coff=12, out_coff=64),
    # 8 x 5000 rows x 128 / 4 = 1.28 M float4 > the 132 * 32 * 256 launch cap: the grid-stride loop wraps
    ew_gate_res_grid_stride=dict(_E, mode='GATE_RES', B=8, T=5000, C=128, gate=True, res=True, act2=L.ACT_RELU),
    ew_aff_grid_stride=dict(_E, mode='AFF', B=8, T=5000, C=128, saturate=True),
    ew_copy_window=dict(_E, mode='COPY', B=3, T=97, C=36, in_coff=4, out_coff=8),
    pad_copy_c201=dict(op='ew', kernel='pad_copy', mode='PAD_COPY', B=3, T=97, C=201, Cout=204, in_coff=1),
    pad_copy_c257=dict(op='ew', kernel='pad_copy', mode='PAD_COPY', B=2, T=151, C=257, Cout=260, in_coff=3,
                       out_coff=4),
    # softmax over T with logits around +80 / +200: exp() only stays finite after the max subtraction
    asp_logits_plus80=dict(op='asp', kernel='asp_smem', B=3, R=298, C=72, logit_shift=80.0),
    asp_logits_plus200_global=dict(op='asp', kernel='asp', B=3, R=900, C=72, logit_shift=200.0),
    asp_c36=dict(op='asp', kernel='asp_smem', B=3, R=298, C=36),
    sap_c36_global=dict(op='asp', kernel='asp', B=3, R=801, C=36, mean_only=True),
    # near-constant columns (mean 1e3, spread 1e-3): a one-pass E[x^2] - E[x]^2 loses every digit, the two-pass
    # centred sum keeps them
    colstats_near_const=dict(op='colstats', kernel='colstats_smem', stats='MEAN_STD_UNBIASED', B=3, R=800, C=72,
                             fill=('normal', 1e-3, 1e3)),
    colstats_near_const_global=dict(op='colstats', kernel='colstats', stats='MEAN_VAR_UNBIASED', B=3, R=1201, C=72,
                                    fill=('normal', 1e-3, 1e3)),
    colstats_c36=dict(op='colstats', kernel='colstats_smem', stats='MEAN_STD_CLAMP', B=3, R=298, C=36),
    colstats_c36_global=dict(op='colstats', kernel='colstats', stats='MEAN_STD_TSTP', B=3, R=1000, C=36),
    # segment context whose last segment holds one row (shared-memory segment sums, and the two-sweep path > 64)
    seg_context_last_one_row=dict(op='colstats', kernel='colstats', stats='SEG_CONTEXT', B=3, R=61, C=72, seg_len=10),
    seg_context_last_one_row_71=dict(op='colstats', kernel='colstats', stats='SEG_CONTEXT', B=2, R=701, C=36,
                                     seg_len=10),
)
# pooling on both sides of each shared-memory limit, C = 72.  ASP / mean-only SAP: both [T, 32] strips are staged up to
# T = 800 (T * 256 B <= 200 KB)
for _T in (400, 401, 800, 801):
    _k = 'asp_smem' if _T <= 800 else 'asp'
    GLUE_CASES[f'asp_T{_T}'] = dict(op='asp', kernel=_k, B=3, R=_T, C=72)
    GLUE_CASES[f'sap_mean_T{_T}'] = dict(op='asp', kernel=_k, B=3, R=_T, C=72, mean_only=True)
# colstats: the [R, 32] strip is staged up to R = 800 rows (R * 128 B <= 100 KB)
for _stats in ('MEAN', 'MEAN_STD_CLAMP', 'MEAN_STD_UNBIASED', 'MEAN_STD_TSTP', 'MEAN_VAR_UNBIASED'):
    for _R in (800, 801):
        GLUE_CASES[f'colstats_{_stats.lower()}_R{_R}'] = dict(op='colstats', kernel='colstats_smem' if _R <= 800
                                                              else 'colstats', stats=_stats, B=3, R=_R, C=72)
# segment context: the segment sums are parked in shared memory up to 64 segments, two sweeps above
for _n in (64, 65):
    GLUE_CASES[f'seg_context_{_n}'] = dict(op='colstats', kernel='colstats', stats='SEG_CONTEXT', B=3, R=10 * _n - 5,
                                           C=72, seg_len=10)
# views that start one column into their matrix: no 16-byte staging, the global-memory kernels run
GLUE_CASES['asp_unaligned_coff'] = dict(op='asp', kernel='asp', B=3, R=298, C=72, in_coff=1)
GLUE_CASES['colstats_unaligned_coff'] = dict(op='colstats', kernel='colstats', stats='MEAN_STD_CLAMP', B=3, R=298, C=72,
                                             in_coff=1)
for _i, _c in enumerate(GLUE_CASES.values()):
    _c['seed'] = 300 + _i

# ---- fp16-split range safety: every writer kernel reports max|y| into the amax slot its TC16 consumer scales by ----
_CONSUMER = dict(B=4, T=300, N=128)                            # 1x1 TC16 conv over the writer's 1200 rows
AMAX_WRITERS = dict(
    ew_gate_res=dict(op='ew', mode='GATE_RES', B=4, T=300, C=64, gate=True, res=True, act2=L.ACT_RELU, out_C=64),
    ew_aff=dict(op='ew', mode='AFF', B=4, T=300, C=64, out_C=64),
    pad_copy=dict(op='ew', mode='PAD_COPY', B=4, T=300, C=201, Cout=208, in_coff=1, out_C=208),
    pool2d=dict(op='pool2d', mode='avg', B=4, Tin=30, Fin=10, C=16, stride=1, out_C=16),
    c1_wide=dict(op='c1', Cin=1, B=4, Tin=30, Fin=10, N=16, KT=3, KF=3, padT=1, padF=1, bias=True, out_C=16),
    c1_generic=dict(op='c1', Cin=1, B=4, Tin=30, Fin=10, N=8, KT=3, KF=3, padT=1, padF=1, bias=True, out_C=8),
    ffma_conv=dict(op='conv', engine='ffma', B=4, Tin=300, Cin=64, N=64, KT=3, padT=1, bias=True, out_C=64),
    tf32_conv=dict(op='conv', engine='tc', B=4, Tin=300, Cin=64, N=64, KT=3, padT=1, bias=True, out_C=64),
    tc16_conv=dict(op='conv', engine='tc16', B=4, Tin=300, Cin=64, N=128, KT=3, padT=1, bias=True, out_C=128),
)
AMAX_KERNELS = dict(ew_gate_res='ew', ew_aff='ew', pad_copy='pad_copy', pool2d='pool2d', c1_wide='conv_c1_wide',
                    c1_generic='conv_c1', ffma_conv='conv_ffma<64>', tf32_conv='conv_tc<tf32>',
                    tc16_conv='conv_tc<f16>', small_m_1024='linear_small_m')
RANGE_SCALES = (1e-30, 1e-6, 1e6, 1e30)
# the scale multiplies every input AND the writers' biases, so the tensor the consumer reads is O(scale) at both ends
# of the sweep (an unscaled bias of ~0.1 would run the small-scale half at unit scale)
AMAX_CASES = {}
for _i, (_name, _w) in enumerate(AMAX_WRITERS.items()):
    for _s in RANGE_SCALES:
        AMAX_CASES[f'{_name}-{_s:g}'] = dict(_w, seed=400 + _i, scale=_s, bias_scale=_s, kernel=AMAX_KERNELS[_name],
                                             consumer=_CONSUMER)
# linear_small_m at M = 1024: the only M that is both small-M (FFMA) and tensor-core eligible for its consumer
for _s in RANGE_SCALES:
    AMAX_CASES[f'small_m_1024-{_s:g}'] = dict(op='conv', engine='ffma', B=4, Tin=256, Cin=64, N=64, bias=True, out_C=64,
                                              seed=420, scale=_s, bias_scale=_s, kernel='linear_small_m',
                                              consumer=dict(B=4, T=256, N=128))
# two writers into column windows of ONE allocation at scales 1e6 (FFMA conv) and 1 (EW residual add), one consumer
# reading all of it: the shared slot must hold the larger maximum whichever op writes last
_BIG = dict(op='conv', engine='ffma', B=4, Tin=300, Cin=64, N=64, KT=3, padT=1, bias=True, out_C=64, xscale=1e6)
_SMALL = dict(op='ew', mode='GATE_RES', B=4, T=300, C=64, res=True, out_C=64)
SHARED_SLOT_CASES = {
    'big_first': dict(op='conv', B=4, seed=430, consumer=_CONSUMER, windows=[_BIG, _SMALL]),
    'small_first': dict(op='conv', B=4, seed=431, consumer=_CONSUMER, windows=[_SMALL, _BIG]),
}

# slot reset between graph replays: EW copy -> TC16 conv, run at 1e30, then at 1e-30 through the captured graph
GRAPH_RESET = dict(op='ew', mode='COPY', B=4, T=300, C=64, out_C=64, seed=440, kernel='ew', consumer=_CONSUMER)

# one 512 x 512 GEMM over 8 x 298 rows (EW copy -> TC16 conv) at input scales 1e-30 ... 1e30: the fp16 split neither
# overflows (|x| > 65504) nor loses small tensors to fp16 subnormals, its error does not depend on the magnitude
TC16_RANGE_CASES = {f'gemm_512-{_s:g}': dict(op='ew', mode='COPY', B=8, T=298, C=512, out_C=512, seed=450, scale=_s,
                                             kernel='ew', consumer=dict(B=8, T=298, N=512))
                    for _s in (1e-30, 1e-8, 1e-3, 1e4, 1e9, 1e30)}
