"""CPU checks of the op-level edge cases (tests/op_cases.py), no GPU needed:

* the interpreter the GPU tests compare against (tests/plan_sim.py) agrees, case by case, with an independent fp64
  torch evaluation of the same program -- F.conv2d over an explicit reflect / zero F.pad, F.max_pool2d /
  F.avg_pool2d(count_include_pad=True), softmax-weighted statistics, torch.var, the AFF formula;
* coverage intent: every case reaches the kernel it names (the launchers' predicates, mirrored with their source lines
  in op_cases.kernel_of / tc_schedule) on the engine it requests, the tile / chunk schedules the tables claim, and the
  amax slots the fp16 split relies on;
* the engine requests the library refuses (op_cases.REFUSED_CASES) are refused by the engine mirror
  (op_cases.engine_of)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import op_cases as oc
from mvector import _lib as L

ALL = {**{f'tc/{k}': v for k, v in oc.TC_CASES.items()}, **{f'engine/{k}': v for k, v in oc.ENGINE_CASES.items()},
       **{f'ffma/{k}': v for k, v in oc.FFMA_CASES.items()},
       **{f'glue/{k}': v for k, v in oc.GLUE_CASES.items()}, **{f'amax/{k}': v for k, v in oc.AMAX_CASES.items()},
       **{f'shared/{k}': v for k, v in oc.SHARED_SLOT_CASES.items()}, 'graph/reset': oc.GRAPH_RESET,
       **{f'range/{k}': v for k, v in oc.TC16_RANGE_CASES.items()},
       **{f'wide/{k}': v for k, v in oc.TC16_WIDE_CASES.items()}}
SCALED = {**oc.AMAX_CASES, **oc.TC16_RANGE_CASES}


# ---------------------------------------------------------------------------------------------------------------
# independent fp64 torch evaluation of a lowered program
# ---------------------------------------------------------------------------------------------------------------
def _t_act(v, a):
    return {L.ACT_RELU: torch.relu, L.ACT_HARDTANH20: lambda x: x.clamp(0, 20), L.ACT_SIGMOID: torch.sigmoid,
            L.ACT_TANH: torch.tanh, L.ACT_SILU: F.silu}.get(a, lambda x: x)(v)


class TorchRef:
    def __init__(self, b):
        self.b = b
        self.mem = {L.BUF_INPUT: torch.from_numpy(b.X.astype(np.float64).reshape(-1)),
                    L.BUF_OUTPUT: torch.full((b.pb.out_floats,), float('nan'), dtype=torch.float64)}
        self.ws = torch.full((max(b.pb.peak, 256) // 4,), float('nan'), dtype=torch.float64)
        self.blob = torch.from_numpy(b.blob.astype(np.float64))

    def _buf(self, off):
        return (self.mem[off], 0) if off in self.mem else (self.ws, off // 4)

    def rd(self, off, rows, ld, coff, C):
        mem, base = self._buf(off)
        return mem.as_strided((rows, C), (ld, 1), base + coff).clone()

    def wr(self, off, rows, ld, coff, C, v):
        mem, base = self._buf(off)
        mem.as_strided((rows, C), (ld, 1), base + coff).copy_(v.to(torch.float32).to(torch.float64))

    def w(self, off, n):
        return self.blob[off // 4: off // 4 + n]

    def run(self):
        for o in self.b.pb.ops:
            {L.OP_CONV: self.conv, L.OP_CONV_C1: self.conv, L.OP_COLSTATS: self.colstats, L.OP_ASP_POOL: self.asp,
             L.OP_EW: self.ew, L.OP_POOL2D: self.pool2d}[o.kind](o)
        return self.mem[L.BUF_OUTPUT].numpy().reshape(self.b.out_rows, self.b.out_cols)

    def conv(self, o):
        B, M = o.B, o.B * o.Tout * o.Fout
        cin = o.Cin + (o.Cin2 if o.src2_mode == L.SRC2_CONCAT else 0)
        x = self.rd(o.src, B * o.Tin * o.Fin, o.in_ld, o.in_coff, o.Cin)
        if o.src2_mode == L.SRC2_ADD:
            x = x + self.rd(o.src2, B * o.Tin * o.Fin, o.src2_ld, o.src2_coff, o.Cin)
        elif o.src2_mode == L.SRC2_CONCAT:
            x = torch.cat([x, self.rd(o.src2, B * o.Tin * o.Fin, o.src2_ld, o.src2_coff, o.Cin2)], 1)
        if o.pre_s >= 0:
            x = x * self.w(o.pre_s, cin) + self.w(o.pre_h, cin)
            x = torch.relu(x) if o.pre_relu else x
        x = x.reshape(B, o.Tin, o.Fin, cin).permute(0, 3, 1, 2)
        if o.pad_mode == L.PAD_REFLECT:
            x = F.pad(x, (0, 0, o.padT, o.padT), mode='reflect')
        else:
            x = F.pad(x, (o.padF, o.padF, o.padT, o.padT))
        K = o.KT * o.KF * cin
        W = self.blob[o.w // 4:o.w // 4 + o.Cout * o.w_ld].reshape(o.Cout, o.w_ld)[:, :K]
        W = W.reshape(o.Cout, o.KT, o.KF, cin).permute(0, 3, 1, 2)
        y = F.conv2d(x, W, stride=(o.sT, o.sF), dilation=(o.dT, o.dF))[:, :, :o.Tout, :o.Fout]
        assert y.shape[2:] == (o.Tout, o.Fout)
        y = y.permute(0, 2, 3, 1)                                         # [B, Tout, Fout, N]
        seg = (torch.arange(o.Tout) // o.seg_len).clamp(max=o.n_seg - 1)

        def per_utt(off):                                                # [B * n_seg, N] -> [B, Tout, 1, N]
            return self.rd(off, B * o.n_seg, o.Cout, 0, o.Cout).reshape(B, o.n_seg, o.Cout)[:, seg, None]

        if o.bias >= 0:
            y = y + self.w(o.bias, o.Cout)
        if o.ubias != L.BUF_NONE:
            y = y + per_utt(o.ubias)
        y = _t_act(y, o.act)
        if o.post_s >= 0:
            y = y * self.w(o.post_s, o.Cout) + self.w(o.post_h, o.Cout)
        if o.gate != L.BUF_NONE:
            y = y * per_utt(o.gate)
        y = y.reshape(M, o.Cout)
        if o.res != L.BUF_NONE:
            y = y + self.rd(o.res, M, o.res_ld, o.res_coff, o.Cout)
        y = _t_act(y, o.act2)
        self.wr(o.dst, M, o.out_ld, o.out_coff, o.Cout, y)
        if o.sum != L.BUF_NONE:
            self.wr(o.sum, M, o.sum_ld, o.sum_coff, o.Cout, self.rd(o.sum, M, o.sum_ld, o.sum_coff, o.Cout) + y)

    def pool2d(self, o):
        x = self.rd(o.src, o.B * o.Tin * o.Fin, o.in_ld, o.in_coff, o.Cin).reshape(o.B, o.Tin, o.Fin, o.Cin)
        x = x.permute(0, 3, 1, 2)
        args = dict(kernel_size=(o.KT, o.KF), stride=(o.sT, o.sF), padding=(o.padT, o.padF))
        y = F.max_pool2d(x, **args) if o.mode == L.POOL_MAX else F.avg_pool2d(x, count_include_pad=True, **args)
        assert y.shape[2:] == (o.Tout, o.Fout)
        self.wr(o.dst, o.B * o.Tout * o.Fout, o.out_ld, o.out_coff, o.Cin, y.permute(0, 2, 3, 1).reshape(-1, o.Cin))

    def ew(self, o):
        rows = o.B * o.Tin * o.Fin
        x = self.rd(o.src, rows, o.in_ld, o.in_coff, o.Cin)
        if o.mode == L.EW_PAD_COPY:
            self.wr(o.dst, rows, o.out_ld, o.out_coff, o.Cout, F.pad(x, (0, o.Cout - o.Cin)))
            return
        if o.mode == L.EW_GATE_RES:
            if o.gate != L.BUF_NONE:
                x = (x.reshape(o.B, -1, o.Cin) * self.rd(o.gate, o.B, o.Cin, 0, o.Cin)[:, None]).reshape(rows, o.Cin)
            if o.res != L.BUF_NONE:
                x = x + self.rd(o.res, rows, o.res_ld, o.res_coff, o.Cin)
            x = _t_act(x, o.act2)
        elif o.mode == L.EW_AFF:                        # eres2net.py AFF: x * (1 + tanh(a)) + y * (1 - tanh(a))
            y = self.rd(o.src2, rows, o.src2_ld, o.src2_coff, o.Cin)
            t = torch.tanh(self.rd(o.res, rows, o.res_ld, o.res_coff, o.Cin))
            x = x * (1 + t) + y * (1 - t)
        self.wr(o.dst, rows, o.out_ld, o.out_coff, o.Cin, x)

    def colstats(self, o):
        R = o.Tin * o.Fin
        x = self.rd(o.src, o.B * R, o.in_ld, o.in_coff, o.Cin).reshape(o.B, R, o.Cin)
        mean = x.mean(1)
        if o.mode == L.STATS_MEAN:
            out = mean
        elif o.mode == L.STATS_SEG_CONTEXT:
            segs = torch.split(x, o.seg_len, dim=1)
            assert len(segs) == o.n_seg
            out = torch.stack([mean + s.mean(1) for s in segs], 1).reshape(-1, o.Cin)
        else:
            second = {L.STATS_MEAN_STD_CLAMP: lambda: x.var(1, unbiased=False).clamp(min=o.eps).sqrt(),
                      L.STATS_MEAN_STD_UNBIASED: lambda: x.std(1),
                      L.STATS_MEAN_VAR_UNBIASED: lambda: x.var(1),
                      L.STATS_MEAN_STD_TSTP: lambda: (x.var(1) + o.eps).sqrt()}[o.mode]()
            out = torch.cat([mean, second], 1)
        self.wr(o.dst, out.shape[0], o.out_ld, o.out_coff, out.shape[1], out)

    def asp(self, o):
        x = self.rd(o.src, o.B * o.Tin, o.in_ld, o.in_coff, o.Cin).reshape(o.B, o.Tin, o.Cin)
        a = torch.softmax(self.rd(o.src2, o.B * o.Tin, o.src2_ld, o.src2_coff, o.Cin).reshape(o.B, o.Tin, o.Cin), 1)
        mean = (a * x).sum(1)
        out = mean if o.mode == 1 else torch.cat(
            [mean, (a * (x - mean[:, None]) ** 2).sum(1).clamp(min=o.eps).sqrt()], 1)
        self.wr(o.dst, o.B, o.out_ld, o.out_coff, out.shape[1], out)


def _small(case):
    """The 16-utterance multi-tile cases at B = 2: the same op at an eighth of the rows (the fp64 torch conv is slow)."""
    return oc.with_batch(case, 2) if case.get('B', 1) >= 16 else case


@pytest.mark.parametrize('name', list(ALL))
def test_interpreter_matches_torch(name):
    b = oc.build(_small(ALL[name]))
    ref = TorchRef(b).run()
    got = oc.sim(b)
    assert np.isfinite(ref).all()
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-9 * np.abs(ref).max())


def test_interpreter_matches_torch_on_position_invariance_case():
    for variant in oc.INVARIANCE_VARIANTS:
        b = oc.build(oc.invariance(variant, 'tc', 1))
        np.testing.assert_allclose(oc.sim(b), TorchRef(b).run(), rtol=1e-6, atol=1e-9)


# ---------------------------------------------------------------------------------------------------------------
# coverage intent
# ---------------------------------------------------------------------------------------------------------------
def _main_ops(b):
    return [b.main] if isinstance(b.main, int) else list(b.main)


def _kernel(b, i):
    return oc.kernel_of(b.pb.ops[i], b.expect.get(i, 0))


@pytest.mark.parametrize('name', [n for n in ALL if ALL[n].get('kernel')])
def test_case_reaches_its_kernel(name):
    b = oc.build(ALL[name])
    assert oc.engine_of(b.pb.finalize().ops[b.main]) == b.expect.get(b.main, 0)     # the request is not refused
    assert _kernel(b, b.main) == ALL[name]['kernel']


@pytest.mark.parametrize('name', list(oc.REFUSED_CASES))
def test_engine_mirror_refuses_unsupported_request(name):
    b = oc.build(oc.REFUSED_CASES[name])
    with pytest.raises(ValueError):
        oc.engine_of(b.pb.finalize().ops[b.main])


def _schedules():
    out = {}
    for name, case in oc.TC_CASES.items():
        if case['engine'] == 'ffma':
            continue
        b = oc.build(case)
        out[name] = (case, oc.tc_schedule(b.pb.ops[b.main], b.expect[b.main]))
    return out


SCHED = None


def _sched():
    global SCHED
    if SCHED is None:
        SCHED = _schedules()
    return SCHED


def test_tc_cases_have_the_schedules_they_claim():
    for name, (case, s) in _sched().items():
        for key, want in case.get('intent', {}).items():
            if key == 'chunk_remainder':
                assert s['n_chunks'] > 1 and s['last_chunk'] < s['kc'], (name, s)
            else:
                assert s[key] == want, (name, key, s)


def test_tc_coverage():
    """The plain-source kernels (conv_tc<tf32>, conv_tc<f16>) reach >= 4 tiles per CTA and exactly 133 tiles on both
    tensor-core engines, a chunk remainder under both chunk policies on both, every N-tile width, M tails of one row and
    tiles that all take the fast epilogue.  (The add / prologue families: tests/test_conv_gathers_cpu.py.)"""
    S = {n: (c, s) for n, (c, s) in _sched().items() if c['kernel'] in ('conv_tc<tf32>', 'conv_tc<f16>')}
    for eng in ('tc', 'tc16'):
        mine = {n: s for n, (c, s) in S.items() if c['engine'] == eng}
        assert any(s['tiles_per_cta'] >= 4 for s in mine.values()), eng
        assert any(s['tiles'] == 133 and s['tiles_per_cta'] == 2 for s in mine.values()), eng
        for policy in (oc.ERES_POLICY, oc.DEFAULT_POLICY):
            assert any(S[n][0].get('policy', oc.DEFAULT_POLICY) == policy and s['n_chunks'] > 1
                       and s['last_chunk'] < s['kc'] for n, s in mine.items()), (eng, policy)
        assert any(s['m_tail'] == 1 for s in mine.values()), eng
        assert any(s['fast'] for s in mine.values()), eng
    # every wgmma N piece combination of the split-TF32 engine (n16 .. n128 with column tails)
    bns = {s['bn'] for c, s in S.values() if c['engine'] == 'tc'}
    assert {32, 48, 64, 80, 96, 112, 128} <= bns, bns
    # K = 2304 at 8-block (tf32) and 4-block (f16) chunks
    k2304 = {c['engine']: s['kc'] for c, s in S.values() if c.get('Cin') == 256 and c.get('KT') == 3}
    assert k2304 == {'tc': 8, 'tc16': 4}, k2304


def _wide_schedules():
    out = {}
    for name, case in oc.TC16_WIDE_CASES.items():
        if case['kernel'] == 'conv_tc16_wide':
            b = oc.build(case)
            out[name] = (case, b.pb.ops[b.main], oc.wide_schedule(b.pb.ops[b.main]))
    return out


def test_tc16_wide_cases_have_the_schedules_they_claim():
    for name, (case, _, s) in _wide_schedules().items():
        for key, want in case.get('intent', {}).items():
            assert s[key] == want, (name, key, s)


def test_tc16_wide_coverage():
    """The wide kernel's edges: several tiles per CTA with an odd K-block count and a residual (the 2-stage ring's
    phase carried across tiles, the next tile's residual prefetched), exactly 133 tiles, an M tail of one row, K < 64
    in one partial block, K = 64 in one full block, a K tail after full blocks, M = 1024, input and output column
    windows, and every epilogue feature (residual, affine, ubias, per-segment gate, accumulate-into, SiLU / sigmoid /
    tanh)."""
    W = {n: (o, s) for n, (_, o, s) in _wide_schedules().items()}
    sched = [s for _, s in W.values()]
    assert any(s['tiles_per_cta'] >= 2 and s['k_blocks'] % 2 == 1 and s['k_blocks'] > 1 and o.res != L.BUF_NONE
               for o, s in W.values())
    assert any(s['tiles'] == 133 and s['tiles_per_cta'] == 2 for s in sched)
    assert any(s['m_tail'] == 1 for s in sched)
    assert {8, 40} <= {s['K'] for s in sched if s['k_blocks'] == 1 and s['k_tail']}
    assert any(s['K'] == 64 for s in sched)
    assert any(s['k_blocks'] > 1 and s['k_tail'] for s in sched)
    assert min(s['M'] for s in sched) == 1024
    ops = [o for o, _ in W.values()]
    assert any(o.in_coff > 0 for o in ops) and any(o.out_coff > 0 for o in ops)
    assert any(o.gate != L.BUF_NONE and o.n_seg > 1 for o in ops)
    assert any(o.ubias != L.BUF_NONE for o in ops) and any(o.sum != L.BUF_NONE for o in ops)
    assert any(o.post_s >= 0 for o in ops) and any(o.res != L.BUF_NONE for o in ops)
    assert {L.ACT_SILU, L.ACT_SIGMOID, L.ACT_TANH} <= {o.act for o in ops} | {o.act2 for o in ops}


def test_position_invariance_case_lands_on_full_and_tail_tiles():
    for variant, engine in ((v, e) for v in oc.INVARIANCE_VARIANTS for e in ('tc', 'ffma')):
        b16 = oc.build(oc.invariance(variant, engine, 16))
        b3 = oc.build(oc.invariance(variant, engine, 3))
        o16, o3 = b16.pb.ops[b16.main], b3.pb.ops[b3.main]
        assert _kernel(b16, b16.main) == _kernel(b3, b3.main) != 'linear_small_m'
        if engine == 'tc':
            s16, s3 = oc.tc_schedule(o16, L.ENGINE_TC), oc.tc_schedule(o3, L.ENGINE_TC)
            assert s16['fast'] and s16['tiles_per_cta'] >= 4
            assert s3['simple'] and s3['m_tail'] != 0 and s3['bn'] == s16['bn']     # full tiles fast, the tail general
        else:
            assert (o16.B * o16.Tout) % 128 == 0 and (o3.B * o3.Tout) % 128 != 0


def test_every_kernel_is_reached():
    reached = set()
    for case in ALL.values():
        b = oc.build(_small(case))
        reached |= {_kernel(b, i) for i in _main_ops(b)}
    want = {'conv_tc<tf32>', 'conv_tc<tf32,add>', 'conv_tc<tf32,pre>', 'conv_tc<f16>', 'conv_tc16_wide', 'conv_ffma<32>',
            'conv_ffma<64>', 'conv_ffma<128>', 'linear_small_m', 'conv_c1_wide', 'conv_c1', 'pool2d', 'ew', 'pad_copy',
            'colstats', 'colstats_smem', 'asp', 'asp_smem'}
    assert want <= reached, want - reached


def test_small_m_dimensions_are_covered():
    Ms, Ks, Ns = set(), set(), set()
    for case in oc.FFMA_CASES.values():
        b = oc.build(case)
        o = b.pb.ops[b.main]
        M = o.B * o.Tout * o.Fout
        if _kernel(b, b.main) == 'linear_small_m':
            Ms.add(M)
            Ks.add(o.KT * o.KF * o.Cin)
            Ns.add(o.Cout)
        else:
            assert M > 1024 or o.KT * o.KF > 1 or o.kind == L.OP_CONV_C1
    assert {1, 7, 8, 9, 1023, 1024} <= Ms and {4, 124, 128, 132, 3072} <= Ks and {4, 28, 36, 192} <= Ns
    b = oc.build(oc.FFMA_CASES['tiled_m1025'])
    assert not oc.small_m_ok(b.pb.ops[b.main])


def test_glue_grid_stride_and_windows():
    strided = []
    for n, c in oc.GLUE_CASES.items():
        b = oc.build(c)
        if b.pb.ops[b.main].kind in (L.OP_EW, L.OP_POOL2D) and oc.ew_grid_strides(b.pb.ops[b.main]):
            strided.append(n)
    assert {'ew_gate_res_grid_stride', 'ew_aff_grid_stride'} <= set(strided), strided
    for name in ('pool_avg_s2_window', 'ew_gate_res_window', 'ew_aff_window', 'pad_copy_c257'):
        b = oc.build(oc.GLUE_CASES[name])
        o = b.pb.ops[b.main]
        assert o.out_coff > 0 and o.out_ld > o.out_coff + (o.Cout if o.mode == L.EW_PAD_COPY and o.kind == L.OP_EW
                                                           else o.Cin), name


@pytest.mark.parametrize('name', [n for n in ALL if 'consumer' in ALL[n]])
def test_amax_slots_link_writer_and_consumer(name):
    """PlanBuilder.finalize gives the TC16 consumer an amax_in slot and every writer of its source allocation the
    matching amax_out."""
    b = oc.build(ALL[name])
    b.pb.finalize()
    consumer = b.pb.ops[b.consumer]
    assert consumer.amax_in > 0 and b.expect[b.consumer] == L.ENGINE_TC16
    for i in _main_ops(b):
        assert b.pb.ops[i].amax_out == consumer.amax_in, (name, i)


@pytest.mark.parametrize('name', list(SCALED))
def test_amax_consumer_sees_the_scale(name):
    """At every scale of the sweep, the tensor the TC16 consumer reads -- and hence its output -- is O(scale): nothing
    unscaled (a bias, a residual) pulls the small-scale cases back to unit magnitude."""
    case = SCALED[name]
    peak = np.abs(oc.sim(oc.build(case))).max() / case['scale']
    assert 1e-2 <= peak <= 1e3, peak


def test_amax_writers_cover_every_writer_kernel():
    kernels = {oc.AMAX_KERNELS[n.split('-')[0]] for n in oc.AMAX_CASES}
    assert kernels == {'ew', 'pad_copy', 'pool2d', 'conv_c1_wide', 'conv_c1', 'conv_ffma<64>', 'linear_small_m',
                       'conv_tc<tf32>', 'conv_tc<f16>', 'conv_tc16_wide'}
    scales = {c['scale'] for c in oc.AMAX_CASES.values()}
    assert scales == set(oc.RANGE_SCALES)
    b = oc.build(oc.AMAX_CASES['small_m_1024-1e+06'])
    assert b.pb.ops[b.consumer].B * b.pb.ops[b.consumer].Tout == 1024
