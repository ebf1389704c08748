"""CPU checks of the add / prologue gather cases of tests/op_cases.py and of the tensor-core kernels the benchmark
configurations reach, no GPU needed:

* every tensor-core kernel instantiation (family, N tile, chunked or not) that a bench.py configuration runs -- on the
  engines op_cases.engine_of resolves, with the fp16 split on and off -- is among the schedules of TC_CASES, so a model
  change that reaches a new instantiation fails here until a case covers it;
* the add and prologue families each reach the schedules and geometries their gathers branch on;
* the MODE 0 twins the GPU compares against are what they claim to be."""
import numpy as np
import pytest

import op_cases as oc
from mvector import _lib as L

FAMILY = {'add': 'conv_tc<tf32,add>', 'pre': 'conv_tc<tf32,pre>'}
_CACHE = {}


def _tc_cases():
    """name -> (case, op, schedule) for every TC_CASES entry on a tensor-core engine."""
    if 'tc' not in _CACHE:
        out = {}
        for name, case in oc.TC_CASES.items():
            if case['engine'] != 'ffma':
                b = oc.build(case)
                o = b.pb.ops[b.main]
                out[name] = (case, o, oc.tc_schedule(o, b.expect[b.main]), oc.kernel_of(o, b.expect[b.main]))
        _CACHE['tc'] = out
    return _CACHE['tc']


def _reach(o, engine):
    s = oc.tc_schedule(o, engine)
    return oc.kernel_of(o, engine), s['bn'], s['n_chunks'] > 1


@pytest.mark.parametrize('cfg', sorted(oc.BENCH_T))
def test_product_tensor_core_kernels_are_covered(cfg):
    """Lowered at the bench batch and T.  With the fp16 split off (VPB_TC_F16=0), AUTO sends its MODE 0 layers to
    split TF32 at the same N tile: both routings must be covered."""
    model, c = oc.bench_model(cfg)
    pb = model.lower(c['per_gpu'], oc.BENCH_T[cfg]).finalize()
    have = {_reach(o, oc.ENGINES[c['engine']]) for c, o, _, _ in _tc_cases().values()}
    reach = set()
    for tc16_on in (True, False):
        for o in pb.ops:
            e = oc.engine_of(o, tc16_on=tc16_on)
            if e in (L.ENGINE_TC, L.ENGINE_TC16):
                reach.add(_reach(o, e))
    assert reach, cfg
    assert reach <= have, sorted(reach - have)


def _family(fam):
    return {n: v for n, v in _tc_cases().items() if v[3] == FAMILY[fam]}


@pytest.mark.parametrize('fam', sorted(FAMILY))
def test_family_coverage(fam):
    """The schedules of each gather family: every N tile (composite ones with a column tail), a chunk remainder under the
    policy the family's models use, >= 4 tiles per CTA and exactly 133 tiles on 132 CTAs, a one-row M tail, a K tail,
    one K block per tile with several tiles per CTA and an odd item count, all tiles on the fast epilogue, and the
    general epilogue through a feature rather than a tail."""
    F = _family(fam)
    S = [s for _, _, s, _ in F.values()]
    assert {16, 32, 48, 64, 80, 96, 112, 128} <= {s['bn'] for s in S}
    for bn in (48, 80, 96, 112):
        assert any(s['bn'] == bn and o.Cout % bn for _, o, s, _ in F.values()), bn
    policy = oc.ERES_POLICY if fam == 'add' else oc.DEFAULT_POLICY
    assert any(c.get('policy', oc.DEFAULT_POLICY) == policy and s['n_chunks'] > 1 and s['last_chunk'] < s['kc']
               for c, _, s, _ in F.values())
    assert any(s['tiles_per_cta'] >= 4 for s in S)
    assert any(s['tiles'] == 133 and s['tiles_per_cta'] == 2 for s in S)
    assert any(s['m_tail'] == 1 for s in S)
    assert any(s['k_tail'] for s in S)
    assert any(s['k_blocks'] == 1 and s['tiles_per_cta'] > 1 and s['items'] % 2 for s in S)
    assert any(s['fast'] for s in S)
    assert any(not s['simple'] for s in S)
    # every case also runs on the FFMA engine (the same gather semantics, exact fp32)
    strip = lambda c: {k: v for k, v in c.items() if k not in ('engine', 'kernel')}
    for name, (c, _, _, _) in F.items():
        assert strip(oc.TC_CASES.get(name[:-len('-tc')] + '-ffma', {})) == strip(c), name


def test_add_geometries():
    """Reflect padding at the smallest map for dilations 2, 3, 4; a zero-padded 3x3 map with odd Fin; a second source
    in its own allocation with another row pitch and another first column."""
    ops = [o for _, o, _, _ in _family('add').values()]
    for d in (2, 3, 4):
        assert any(o.pad_mode == L.PAD_REFLECT and o.dT == d and o.padT == d and o.KT == 3 and o.Tin == d + 1
                   for o in ops), d
    assert any(o.KT == 3 and o.KF == 3 and o.pad_mode == L.PAD_ZERO and o.padF > 0 and o.Fin % 2 for o in ops)
    assert any(o.src2 >= 0 and o.src2_ld != o.in_ld and o.src2_coff != o.in_coff for o in ops)


def test_prologue_geometries():
    """A column window of a wider map (in_ld > Cin), zero padding with KT = 3 and with 3x3, reflect padding, no ReLU,
    and CAM++'s last transit (N = 512, K = 1024, BN affine + ReLU after the conv)."""
    ops = [o for _, o, _, _ in _family('pre').values()]
    assert all(o.pre_s >= 0 for o in ops)
    assert any(o.in_ld > o.Cin and o.in_coff > 0 for o in ops)
    assert any(o.KT == 3 and o.KF == 1 and o.padT > 0 and o.pad_mode == L.PAD_ZERO for o in ops)
    assert any(o.KT == 3 and o.KF == 3 and o.padF > 0 and o.pad_mode == L.PAD_ZERO for o in ops)
    assert any(o.pad_mode == L.PAD_REFLECT and o.padT > 0 for o in ops)
    assert any(not o.pre_relu for o in ops)
    assert any(o.Cout == 512 and o.KT * o.KF * o.Cin == 1024 and o.post_s >= 0 and o.act2 == L.ACT_RELU for o in ops)


@pytest.mark.parametrize('name', list(oc.GATHER_CASES))
def test_twin_is_the_plain_gather_of_the_same_operand(name):
    """The twin keeps weights, geometry, schedule and epilogue and only swaps the gather: its fp64 reference differs
    from the original's by the fp32 rounding of the operand alone.  Its operand is, element by element, the float the
    kernels' fp32 add / fmaf yields (checked here against fp32 arithmetic for the add, and for the prologue against the
    exact product x * s, which the power-of-two scales keep in fp32)."""
    case = oc.GATHER_CASES[name]
    b, t = oc.build(case), oc.build(oc.twin(case))
    o, ot = b.pb.ops[b.main], t.pb.ops[t.main]
    assert ot.src2_mode == L.SRC2_NONE and ot.pre_s < 0 and ot.engine == o.engine
    for f in ('w', 'w_tc', 'tc_bn', 'tc_kc', 'Cout', 'KT', 'KF', 'dT', 'padT', 'padF', 'pad_mode', 'Tin', 'Fin', 'B',
              'bias', 'post_s', 'act', 'act2'):
        assert getattr(ot, f) == getattr(o, f), f
    e = b.expect[b.main]
    assert t.expect[t.main] == e and oc.kernel_of(ot, e) == case['kernel'].replace(',add', '').replace(',pre', '')
    if e == L.ENGINE_TC:
        assert oc.tc_schedule(ot, e) == oc.tc_schedule(o, e)
    rows = o.B * o.Tin * o.Fin
    assert o.src == ot.src == L.BUF_INPUT and ot.in_coff >= b.X.shape[1]
    x = b.X[:rows, o.in_coff:o.in_coff + o.Cin]
    op = t.X[:rows, ot.in_coff:ot.in_coff + ot.Cin]
    np.testing.assert_array_equal(t.X[:, :b.X.shape[1]], b.X)          # the twin's other inputs are the original's
    if o.pre_s >= 0:
        s = b.blob[o.pre_s // 4:o.pre_s // 4 + o.Cin]
        assert np.array_equal((x * s).astype(np.float64), x.astype(np.float64) * s)        # x * s exact in fp32
        d = (x * s).astype(np.float64) + b.blob[o.pre_h // 4:o.pre_h // 4 + o.Cin]
        want = d.astype(np.float32)
        np.testing.assert_array_equal(op, np.maximum(want, 0) if o.pre_relu else want)
    else:
        # y: the input columns of the second source, or those its own allocation was copied from
        ycol = o.src2_coff if o.src2 == L.BUF_INPUT else next(p.in_coff for p in b.pb.ops if p.dst == o.src2)
        np.testing.assert_array_equal(op, x + b.X[:rows, ycol:ycol + o.Cin])
    ref, ref_t = oc.sim(b), oc.sim(t)
    assert np.abs(ref - ref_t).max() <= 1e-5 * max(1.0, np.abs(ref).max())
