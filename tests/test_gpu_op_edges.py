"""Op-level GPU tests at the shapes and edges where the backbone kernels go wrong: the persistent tensor-core schedule
(several tiles per CTA, 133 tiles on 132 SMs), M / N / K tails, accumulation-chunk remainders, reflect padding at the
smallest map, the fp16 split's epilogues, the backbones' conv geometries on every engine and the engine AUTO picks, the
FFMA family (small-M linear, tiled conv, both 2-D stem kernels), the glue kernels (pool2d, ew, pad copy, colstats, ASP,
on both sides of their shared-memory limits) and the amax tracking that keeps the fp16 split range-safe.

Each case is one op (plus the copies that feed it) from tests/op_cases.py, compared element by element with the fp64
interpreter (tests/plan_sim.py) against a bound built from the fp32 arithmetic of the kernel that ran it
(tests/error_bound.py): max |got - ref| / beta <= 1, printed as err/beta beside the old flat max-rel metric; max pooling
and copies bit-exact.  Every conv asserts the engine it ran on, so a case cannot pass through a silent fallback, and an
engine request the op cannot take must be refused when the program is created.  Every case also runs as a captured
CUDA graph and as a replay of it on a second input (op_cases.run_gpu), bit-identical to the eager runs.

The program lifecycle tests at the end cover what the graph cache is keyed on: new input / output pointers, the
fall-back to eager runs after 16 misses, an arena reallocated under a captured graph, a weight reload (programs created
before it are refused) and two models sharing one Engine.

The max-rel errors quoted in the docstrings were measured on an H100 80GB HBM3 at 700 W."""
import numpy as np
import pytest
import torch

import error_bound as eb
import op_cases as oc
from mvector import _lib as L

pytestmark = pytest.mark.gpu


_rel = eb.max_rel


def _run(case):
    b = oc.build(case)
    got, ops = oc.run_gpu(b)
    oc.assert_engines(b, ops)
    return b, got, oc.sim(b)


def _gate(name, case, floor=1.0):
    """Run a case and hold every element to its own bound: max |got - ref| / beta <= 1 (the old max-rel printed beside)."""
    b = oc.build(case)
    got, ops = oc.run_gpu(b)
    oc.assert_engines(b, ops)
    ref, beta = eb.bounded(b)
    r = eb.ratio(got, ref, beta)
    print(f'{name}: err/beta {r:.3f}, max-rel err {_rel(got, ref, floor):.2e}')
    assert r <= 1.0, r
    return b, got, ref


@pytest.mark.parametrize('name', list(oc.TC_CASES))
def test_conv_schedule_and_tails(name):
    """Tensor-core engines (and the FFMA reference on the reflect / window / add / prologue cases) on multi-tile
    schedules, M / N / K tails, chunk remainders, fp16-split epilogues and the add / BN-ReLU prologue gathers.  Measured
    max-rel error: split TF32 <= 3.2e-6 on the plain source (largest: K = 1600 chunked by 512), <= 1.9e-6 with the add,
    <= 7.9e-6 with the prologue (CAM++'s transit, K = 1024); fp16 split <= 1.8e-6; FFMA <= 1.2e-6."""
    _gate(name, oc.TC_CASES[name])


@pytest.mark.parametrize('name', list(oc.ENGINE_CASES))
def test_conv_engines_on_backbone_geometries(name):
    """The backbones' conv geometries on exact fp32 FFMA, split TF32 and (N >= 128) the fp16 split, and the engine AUTO
    resolves to where a tensor-core engine cannot take the op (FFMA for a prologue with a second source, split TF32 on
    the raw program input), gated by the engine that ran.  Measured max-rel error: FFMA <= 7.5e-6; split TF32 <= 3.7e-6
    at K <= 512 and up to 4.1e-5 at K = 1536, the longest unchunked accumulation -- the tensor core's fp32 accumulator
    truncates on every accumulate, a bias that does not average out, still 10-100x below single-pass TF32's ~1e-3;
    fp16 split <= 2.2e-5 (K = 1536)."""
    _gate(name, oc.ENGINE_CASES[name])


def test_unsupported_engine_requests_are_refused():
    """An explicit tensor-core request the op cannot take (a prologue with a second source on split TF32, the fp16 split
    on an untracked source) fails when the program is created: never a silently different result."""
    for name, case in oc.REFUSED_CASES.items():
        with pytest.raises(L.VpError):
            oc.run_gpu(oc.build(case))
            pytest.fail(f'{name}: the program was created and ran')


@pytest.mark.parametrize('engine', ['tc', 'ffma', 'add-tc', 'add-ffma', 'pre-tc', 'pre-ffma'])
def test_rows_do_not_depend_on_tile_position(engine):
    """The first three utterances give bit-identical rows at B = 16 (125 full tiles: every tile on the fast epilogue,
    ~8 tiles per CTA) and at B = 3 (a tail tile on the general epilogue): the fast and general epilogues compute the
    same expression, and a CTA's second, third, ... tile reads its own rows.  'add-' / 'pre-': the same op with a
    second source added, or with the BN-ReLU prologue (the tensor-core kernel's MODE 1 / MODE 2 gathers)."""
    variant, engine = engine.rpartition('-')[::2]
    b16 = oc.build(oc.invariance(variant, engine, 16))
    b3 = oc.build(oc.invariance(variant, engine, 3))
    assert b3.X.shape[1] == b16.X.shape[1]
    b3.X = np.ascontiguousarray(b16.X[:b3.X.shape[0]])         # same rows for the same utterances
    got16, ops16 = oc.run_gpu(b16)
    got3, ops3 = oc.run_gpu(b3)
    oc.assert_engines(b16, ops16)
    oc.assert_engines(b3, ops3)
    assert np.isfinite(got16).all() and np.isfinite(got3).all()      # every row stored (the output is NaN-poisoned)
    rows = b3.out_rows
    assert np.array_equal(got16[:rows].view(np.uint32), got3.view(np.uint32))


@pytest.mark.parametrize('name', list(oc.FFMA_CASES))
def test_ffma_family(name):
    """linear_small_m_kernel (M <= 1024), conv_ffma_kernel<32|64|128> with a one-row M tile, the wide and generic 2-D
    stem kernels: exact fp32 FFMA, measured max-rel error <= 1.4e-6 (tanh epilogues; <= 6e-7 without)."""
    _gate(name, oc.FFMA_CASES[name])


EXACT = {'pool_max_k3s1', 'pool_max_k3s2_negative', 'pool_max_fout1_negative', 'ew_copy_window', 'pad_copy_c201',
         'pad_copy_c257'}


@pytest.mark.parametrize('name', list(oc.GLUE_CASES))
def test_glue_kernels(name):
    """pool2d, ew (GATE_RES / AFF / COPY), pad copy, colstats and ASP.  Max pooling and the copies are bit-exact
    (the pad columns exactly +0); the rest within their per-element bound (max-rel measured <= 4.6e-7).  The near-constant
    colstats columns (mean 1e3, spread 1e-3) also check the spread column on its own: the fp32 mean carries an error of
    about one input ulp, which the centred sum of squares sees as a relative variance error of up to ~1e-2 (measured
    7.2e-3 for the std at R = 800, 1.1e-2 for the variance at R = 1201; a one-pass E[x^2] - E[x]^2 is off by 1e5 and
    more)."""
    case = oc.GLUE_CASES[name]
    if name in EXACT:
        b, got, ref = _run(case)
        assert np.array_equal(got, ref)
        if case.get('mode') == 'PAD_COPY':
            c0 = case.get('out_coff', 0) + case['C']
            pad = got[:, c0:c0 + case['Cout'] - case['C']]
            assert not pad.view(np.uint32).any()                 # +0.0 bits, not just == 0
        return
    b, got, ref = _gate(name, case)
    if case.get('fill', ('normal',))[1:] == (1e-3, 1e3):
        C = case['C']
        spread = np.abs(got[:, C:] - ref[:, C:]) / ref[:, C:]
        print(f'{name}: spread column max-rel err {spread.max():.2e}')
        assert spread.max() <= 5e-2, spread.max()


SCALED = {**oc.AMAX_CASES, **oc.TC16_RANGE_CASES}


@pytest.mark.parametrize('name', list(SCALED))
def test_amax_writer_feeds_tc16(name):
    """Every kernel that writes a TC16 source reports max|y| into the source's amax slot: the consumer (1x1 TC16 conv)
    must stay finite and within its bound at input scales 2^-110 ... 2^116 (inputs and writer biases both scaled; the
    ends lie past the +-100 clamp the fp16 split's scale exponent once had), and so must
    a 512 x 512 GEMM over 8 x 298 rows (the gemm_512 cases).  A writer that reports too small a maximum gives the
    consumer too large a scale, and its fp16 hi terms overflow at any magnitude; a writer that reports nothing leaves
    the slot at 0, which means scale 1: overflow at the large scales, flush to zero at the small ones.  (Too large a
    maximum -- an over-reporting writer, a stale slot -- flushes small tensors to zero; see the graph-replay test.)
    Measured max-rel error <= 1.7e-6 (2.3e-6 on the 512 x 512 GEMM, 4.8e-6 behind the wide fp16-split writer, whose
    consumer reduces over K = 1024)."""
    case = SCALED[name]
    b, got, ref = _gate(name, case, floor=0.0)
    assert b.pb.ops[b.consumer].amax_in > 0
    assert np.isfinite(got).all()


@pytest.mark.parametrize('order', list(oc.SHARED_SLOT_CASES))
def test_amax_slot_shared_by_column_windows(order):
    """Two ops write the two column windows of one allocation at scales 1e6 and 1; the TC16 consumer reads all of it.
    Both writers max into one slot, whichever writes last."""
    _, got, _ = _gate(order, oc.SHARED_SLOT_CASES[order], floor=0.0)
    assert np.isfinite(got).all()


def test_amax_slots_reset_between_graph_replays():
    """vp_embed replays a CUDA graph from its second call on; the graph's memset node must zero the amax slots, or a
    1e-30 input run after a 1e30 one is scaled by the stale maximum and flushes to zero in fp16."""
    from mvector.engine import Engine, Program
    big = oc.build(dict(oc.GRAPH_RESET, scale=1e30))
    small = oc.build(dict(oc.GRAPH_RESET, scale=1e-30))
    eng = Engine()
    try:
        eng.load_weights(big.blob)
        prog = Program(eng, big.pb)
        assert oc.program_engines(prog)[big.consumer] == L.ENGINE_TC16
        x = torch.from_numpy(big.X).cuda()
        y = torch.empty(big.out_rows, big.out_cols, device='cuda')
        outs = []
        for X in (big.X, small.X, small.X):               # eager, then captured graph, then graph replay
            x.copy_(torch.from_numpy(X))
            y.fill_(float('nan'))                         # in place (the graph keeps y's pointer): a replay that
            prog.run(x, y)                                # stores nothing must not compare equal to the last run
            outs.append(y.cpu().numpy())
    finally:
        eng.close()
    assert eb.ratio(outs[0], *eb.bounded(big)) <= 1.0
    assert np.isfinite(outs[1]).all() and np.isfinite(outs[2]).all()
    assert eb.ratio(outs[1], *eb.bounded(small)) <= 1.0
    assert np.array_equal(outs[1].view(np.uint32), outs[2].view(np.uint32))


# ---- program lifecycle: the graph cache keyed on (feats, emb, arena), its give-up path, arena growth, weight reloads ----
def _profiled(prog, x, y):
    """Eager run with per-op events (never a graph) -> output on the host."""
    y.fill_(float('nan'))
    prog.run_profiled(x, y)
    return y.cpu().numpy()


def _graphed(prog, x, y):
    y.fill_(float('nan'))
    prog.run(x, y)
    torch.cuda.synchronize()
    return y.cpu().numpy()


def _same(got, want, what):
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f'{what}: {int(bad.sum())} elements differ'


LIFECYCLE = oc.TC_CASES['res_tail-tc16']          # copy -> TC16 conv with residual: an amax slot and the arena


def test_graph_follows_new_pointers():
    """Two inputs and two outputs alternated on one program: every (x, y) pair the graph was not captured for is
    captured anew, and each result equals the eager run on that input bit for bit."""
    from mvector.engine import Engine, Program
    b = oc.build(LIFECYCLE)
    eng = Engine()
    try:
        eng.load_weights(b.blob)
        prog = Program(eng, b.pb)
        xs = [torch.from_numpy(X).cuda() for X in (b.X, oc.second_input(b.X))]
        ys = [torch.empty(b.out_rows, b.out_cols, device='cuda') for _ in range(2)]
        want = [_profiled(prog, x, ys[0]) for x in xs]
        for step in range(10):                    # (x0, y0), (x1, y0), (x0, y1), (x1, y1), ... each pair twice
            i, j = step % 2, (step // 2) % 2
            _same(_graphed(prog, xs[i], ys[j]), want[i], f'step {step}: x{i} -> y{j}')
    finally:
        eng.close()


def test_graph_capture_given_up_after_16_misses():
    """18 distinct (x, y) pairs, all alive, cycled twice: after 16 graph misses the program stops re-capturing and runs
    eagerly (api.cu embed_graph); every result equals the eager run on its input."""
    from mvector.engine import Engine, Program
    b = oc.build(LIFECYCLE)
    eng = Engine()
    try:
        eng.load_weights(b.blob)
        prog = Program(eng, b.pb)
        xs = [torch.from_numpy(np.ascontiguousarray(np.roll(b.X, 7 * k, axis=0))).cuda() for k in range(18)]
        ys = [torch.empty(b.out_rows, b.out_cols, device='cuda') for _ in range(18)]
        want = [_profiled(prog, x, ys[0]) for x in xs]
        for rnd in range(2):
            for k in range(18):
                _same(_graphed(prog, xs[k], ys[k]), want[k], f'round {rnd}, pair {k}')
    finally:
        eng.close()


def test_graph_recaptured_after_arena_growth():
    """Program A is captured; program B (the same weights at ten times the batch) needs a larger workspace, so the
    handle's arena is reallocated; A's graph holds the freed arena and must be re-captured.  A, B, A each equal their
    eager results."""
    from mvector.engine import Engine, Program
    a, big = oc.build(LIFECYCLE), oc.build(oc.with_batch(LIFECYCLE, 40))
    np.testing.assert_array_equal(a.blob, big.blob)
    eng = Engine()
    try:
        eng.load_weights(a.blob)
        pa = Program(eng, a.pb)
        xa, ya = torch.from_numpy(a.X).cuda(), torch.empty(a.out_rows, a.out_cols, device='cuda')
        want_a = _profiled(pa, xa, ya)
        _graphed(pa, xa, ya)                                           # eager
        _same(_graphed(pa, xa, ya), want_a, 'A captured')
        arena = L.lib().vp_workspace_bytes(eng.handle)
        pbig = Program(eng, big.pb)
        assert L.lib().vp_workspace_bytes(eng.handle) > arena
        xb, yb = torch.from_numpy(big.X).cuda(), torch.empty(big.out_rows, big.out_cols, device='cuda')
        want_b = _profiled(pbig, xb, yb)
        _graphed(pbig, xb, yb)                                         # B's eager first run
        _same(_graphed(pa, xa, ya), want_a, 'A after the arena grew')
        _same(_graphed(pbig, xb, yb), want_b, 'B captured')
        _same(_graphed(pa, xa, ya), want_a, 'A replayed')
    finally:
        eng.close()
    assert eb.ratio(want_a, *eb.bounded(a)) <= 1.0


def test_programs_refused_after_weight_reload():
    """A program validated against one weights blob is refused once another is loaded -- run and run_profiled raise
    VP_ERR_INVALID before anything is launched (the output stays NaN) -- rather than replay a graph that reads the freed
    blob with the old blob's offsets and fp16 descales.  A program created after the reload runs on the new blob."""
    from mvector.engine import Engine, Program
    old, new = oc.build(LIFECYCLE), oc.build(dict(oc.GRAPH_RESET))
    assert new.blob.nbytes < old.blob.nbytes                          # the old offsets would overrun the new blob
    eng = Engine()
    try:
        eng.load_weights(old.blob)
        prog = Program(eng, old.pb)
        x, y = torch.from_numpy(old.X).cuda(), torch.empty(old.out_rows, old.out_cols, device='cuda')
        _graphed(prog, x, y)
        _graphed(prog, x, y)                                           # captured
        eng.load_weights(new.blob)
        for what, call in (('run', lambda: prog.run(x, y)), ('run_profiled', lambda: prog.run_profiled(x, y))):
            y.fill_(float('nan'))
            with pytest.raises(L.VpError) as e:
                call()
            assert e.value.code == L.VP_ERR_INVALID, (what, e.value)
            torch.cuda.synchronize()
            assert torch.isnan(y).all(), what
        fresh = Program(eng, new.pb)
        xn, yn = torch.from_numpy(new.X).cuda(), torch.empty(new.out_rows, new.out_cols, device='cuda')
        got = [_graphed(fresh, xn, yn) for _ in range(3)]             # eager, captured, replayed
        _same(got[1], got[0], 'captured')
        _same(got[2], got[0], 'replayed')
    finally:
        eng.close()
    assert eb.ratio(got[0], *eb.bounded(new)) <= 1.0


def test_models_sharing_an_engine(manifest):
    """Two models on one Engine (load_state_dict(..., engine=e)) called alternately: each re-uploads its own blob when
    the other's is resident, and every output equals the same model on a private Engine bit for bit."""
    from conftest import load_golden
    from mvector.engine import Engine
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object

    def model(name, engine=None):
        m, (_, sd) = manifest[name], load_golden(name)
        net = build_model(m['feature_dim'], dict_to_object({'model_conf': {'model': m['model'],
                                                                            'model_args': m['model_args']}}))
        net.load_state_dict({'0.' + k: v for k, v in sd.items()}, engine=engine)
        return net

    names = ('tdnn_small', 'ecapa_small')
    feats = {n: torch.from_numpy(load_golden(n)[0]['feats']).cuda().float().contiguous() for n in names}
    private = {n: model(n) for n in names}
    want = {n: private[n](feats[n]).cpu().numpy() for n in names}
    e = Engine()
    try:
        shared = {n: model(n, engine=e) for n in names}
        for step in range(6):
            n = names[step % 2]
            _same(shared[n](feats[n]).cpu().numpy(), want[n], f'step {step}: {n}')
    finally:
        e.close()
        for m in private.values():
            m.engine.close()
