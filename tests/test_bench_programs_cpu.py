"""CPU checks of the op-by-op program sweep (tests/bench_sweep.py) that tests/test_gpu_bench_programs.py runs on the
bench programs, with the fp64 interpreter (plan_sim.Sim, fp32 storage) in place of the GPU:

* a prefix of a finalized plan keeps every op field, amax slots and resolved engines included;
* on the real bench lowerings, the row sampler reaches every CTA index and tile ordinal of every tensor-core conv and
  every grid-stride pass of every ew / pool2d op;
* the reference of an op on a subset of its rows, from an operand reader, equals the whole-op BoundSim on those rows
  bit for bit, for every op of every op case;
* the whole sweep passes on small lowerings of the four bench models and on the golden small models, and fails on a
  backend that swaps two M tiles, drops a conv's last K block, or splits an fp16 operand at a wrong amax exponent."""
import numpy as np
import pytest

import bench_sweep as bs
import error_bound as eb
import op_cases as oc
from conftest import load_golden
from mvector import _lib as L

BENCH = ['c2', 'c3', 'c4', 'c5']
SMALL_SHAPES = dict(c2=(4, 300), c3=(4, 300), c4=(3, 140), c5=(2, 90))     # B, T: tensor-core convs at M >= 1024
GOLDEN = ['ecapa_small', 'tdnn_small', 'campplus_small', 'resnetse_small', 'eres2net_small', 'res2net_small',
          'eres2netv2_small']


def _bench(name, shape=None):
    model, cfg = oc.bench_model(name)
    B, T = shape or (cfg['per_gpu'], oc.BENCH_T[name])
    return model, model.lower(B, T).finalize()


def _feats(pb, seed=0):
    return np.random.default_rng(seed).standard_normal(pb.in_floats).astype(np.float32)


def _sweep(name, model, pb, feats, mutate=None):
    engines = [oc.engine_of(o) for o in pb.ops]
    blob = np.array(model._blob, dtype=np.float32)                          # the mutations patch their own copy
    return bs.Sweep(name, pb, model._blob, engines, bs.SimBackend(pb, blob, feats, mutate))


@pytest.mark.parametrize('name', BENCH)
def test_prefix_keeps_every_op_field(name):
    model, pb = _bench(name, SMALL_SHAPES[name])
    slots = [(o.amax_in, o.amax_out) for o in pb.ops]
    engines = [oc.engine_of(o) for o in pb.ops]
    assert any(s != (0, 0) for s in slots) or name == 'c3'
    for i in sorted({0, 1, len(pb.ops) // 2, len(pb.ops) - 2, len(pb.ops) - 1}):
        q = bs.prefix(pb, i)
        assert len(q.ops) == len(q._meta) == i + 1
        assert (q.peak, q.in_floats, q.out_floats) == (pb.peak, pb.in_floats, pb.out_floats)
        assert q.finalize() is q                                            # Program keeps the full plan's slots
        for j, o in enumerate(q.ops):
            assert bytes(o) == bytes(pb.ops[j]), (i, j)
            assert (o.amax_in, o.amax_out) == slots[j] and oc.engine_of(o) == engines[j]


@pytest.mark.parametrize('name', BENCH)
def test_sampler_covers_every_cta_ordinal_and_stride(name):
    model, pb = _bench(name)
    rng = np.random.default_rng(0)
    n_tc = n_ew = 0
    for i, o in enumerate(pb.ops):
        e = oc.engine_of(o)
        k = oc.kernel_of(o, e)
        rows = bs.sample_rows(o, e, k, rng)
        M = bs.out_rows(o)
        assert rows.min() >= 0 and rows.max() < M and rows[0] == 0 and rows[-1] == M - 1
        if bs.is_tc(k):
            _, tiles, grid, _ = bs.tc_grid(o, e, k)
            ctas, ords = bs.tc_coverage(o, e, k, rows)
            assert ctas == set(range(grid)) and ords == set(range(-(-tiles // grid))), (name, i, k)
            rpu = o.Tout * o.Fout
            assert set(range(rpu)) | set(range(M - rpu, M)) <= set(rows.tolist())
            n_tc += 1
        elif o.kind in (L.OP_EW, L.OP_POOL2D):
            assert bs.ew_coverage(o, rows) == set(range(bs.ew_passes(o)[0])), (name, i, k)
            n_ew += 1
        elif o.kind in (L.OP_COLSTATS, L.OP_ASP_POOL) or k == 'linear_small_m':
            assert len(rows) == M
    assert n_tc > 0
    print(f'{name}: {len(pb.ops)} ops, {n_tc} tensor-core convs, {n_ew} ew / pool2d')


ALL_CASES = {**oc.TC_CASES, **oc.ENGINE_CASES, **oc.FFMA_CASES, **oc.GLUE_CASES, **oc.TC16_WIDE_CASES,
             **oc.AMAX_CASES, **oc.SHARED_SLOT_CASES, **oc.TC16_RANGE_CASES}


@pytest.mark.parametrize('name', sorted(ALL_CASES))
def test_row_subset_reference_matches_whole_op(name):
    """Every op of the case's program: the reference on a seeded row subset (operands through the reader, the fp16
    exponent passed in) equals the interpreter's whole-op values and bounds on those rows, up to the GEMM's own rounding:
    BLAS may sum a row in another order when M changes, so the fp64 values agree to 2^-40 of the output's magnitude
    (far below any bound) and the bounds, whose fp32 partial sums (chain_abs) carry a 2^-10 margin, to 2^-20."""
    b = oc.build(ALL_CASES[name])
    sim = eb.BoundSim(b.pb, b.blob, b.X)
    rng = np.random.default_rng(len(name))
    for sim.i, o in enumerate(b.pb.ops):
        rd = sim.reader(o)
        M = bs.out_rows(o)
        rows = np.unique(np.concatenate([[0, M - 1], rng.integers(0, M, 37)]))
        s = 0
        if o.kind == L.OP_CONV and sim.engines[sim.i] == L.ENGINE_TC16:
            X, _ = sim._operand(o, rd, np.arange(o.B * o.Tin * o.Fin))
            s = eb.design_scale_exp(np.abs(X).max())
        sub = sim.op(o, rows, rd, s)
        full = sim.op(o)                                                   # stores, as run() does
        if o.kind in (L.OP_COLSTATS, L.OP_ASP_POOL):
            rows = np.arange(M)
        assert sub.keys() == full.keys()
        for key, (v, bnd) in full.items():
            assert np.abs(sub[key][0] - v[rows]).max() <= 2.0 ** -40 * np.abs(v).max(), (name, sim.i, key, 'value')
            assert np.allclose(sub[key][1], bnd[rows], rtol=2.0 ** -20, atol=0), (name, sim.i, key, 'bound')


def _report(name, stats):
    for k, (r, n) in sorted(stats.items()):
        print(f'  {name} {k:20s} err/beta {r:.3f} over {n}')


@pytest.mark.parametrize('name', BENCH)
def test_sweep_passes_on_small_bench_lowerings(name):
    model, pb = _bench(name, SMALL_SHAPES[name])
    sw = _sweep(name, model, pb, _feats(pb))
    stats = sw.run()
    _report(name, stats)
    assert any(bs.is_tc(k) for k in stats)


@pytest.mark.parametrize('name', GOLDEN)
def test_sweep_passes_on_golden_models(name, manifest):
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object
    m = manifest[name]
    z, sd = load_golden(name)
    feats = z['feats']
    model = build_model(feats.shape[2], dict_to_object({'model_conf': {'model': m['model'],
                                                                        'model_args': m['model_args']}}))
    model.load_state_dict(sd)
    pb = model.lower(feats.shape[0], feats.shape[1]).finalize()
    _report(name, _sweep(name, model, pb, feats.reshape(-1)).run())


# ---- mutated backends ----
def _first(pb, pred):
    return next(i for i, o in enumerate(pb.ops) if pred(o, oc.engine_of(o)))


def _tile_swap(target):
    def mutate(be, i, o):
        if i != target:
            return False
        be.sim.conv(o)
        v = eb.views(o)['dst']
        a, b = np.arange(128), np.arange(128, 256)
        mem, ia = be._idx(v, a)
        _, ib = be._idx(v, b)
        mem[ia], mem[ib] = mem[ib].copy(), mem[ia].copy()
        return True
    return mutate


def _k_tail_dropped(target):
    def mutate(be, i, o):
        if i != target:
            return False
        K = o.KT * o.KF * (o.Cin + (o.Cin2 if o.src2_mode == L.SRC2_CONCAT else 0))
        idx = o.w // 4 + np.arange(o.Cout)[:, None] * o.w_ld + np.arange(K - 32, K)[None, :]
        keep = be.sim.blob[idx].copy()
        be.sim.blob[idx] = 0
        be.sim.conv(o)
        be.sim.blob[idx] = keep
        return True
    return mutate


def _wrong_exponent(target, shift):
    """The fp16 split of op ``target``'s source at the design exponent of its true maximum minus ``shift``."""
    def mutate(be, i, o):
        if i != target:
            return False
        v = eb.views(o)['src']
        mem, idx = be._idx(v, np.arange(v[4]))
        x = mem[idx].copy()
        s = eb.design_scale_exp(np.abs(x).max()) - shift
        with np.errstate(over='ignore', invalid='ignore'):
            xs = (x * np.float32(2.0 ** s)).astype(np.float32)
            hi = xs.astype(np.float16).astype(np.float32)
            lo = (xs - hi).astype(np.float16).astype(np.float32)
        mem[idx] = ((hi.astype(np.float64) + lo) * 2.0 ** -s).astype(np.float32)
        be.sim.conv(o)
        mem[idx] = x
        return True
    return mutate


_TC = (L.ENGINE_TC, L.ENGINE_TC16)
MUTATIONS = {                                            # -> the op it targets in a plan
    'tile_swap': (_tile_swap, lambda o, e: e in _TC and o.sum == L.BUF_NONE),
    'k_tail_dropped': (_k_tail_dropped, lambda o, e: e in _TC and o.sum == L.BUF_NONE),
    'wrong_amax_exponent': (lambda t: _wrong_exponent(t, 20), lambda o, e: e == L.ENGINE_TC16),
}


@pytest.mark.parametrize('mutation', list(MUTATIONS))
def test_mutated_backend_fails_the_sweep(mutation):
    model, pb = _bench('c2', SMALL_SHAPES['c2'])
    make, pred = MUTATIONS[mutation]
    target = _first(pb, pred)
    mutate = make(target)
    with pytest.raises(bs.Failure, match=f'op {target} ') as e:
        _sweep('c2', model, pb, _feats(pb), mutate).run()
    print(f'{mutation}: {e.value}')
