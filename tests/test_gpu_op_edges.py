"""Op-level GPU tests at the shapes and edges where the backbone kernels go wrong: the persistent tensor-core schedule
(several tiles per CTA, 133 tiles on 132 SMs), M / N / K tails, accumulation-chunk remainders, reflect padding at the
smallest map, the fp16 split's epilogues, the backbones' conv geometries on every engine and the engine AUTO picks, the
FFMA family (small-M linear, tiled conv, both 2-D stem kernels), the glue kernels (pool2d, ew, pad copy, colstats, ASP,
on both sides of their shared-memory limits) and the amax tracking that keeps the fp16 split range-safe.

Each case is one op (plus the copies that feed it) from tests/op_cases.py, compared with the fp64 interpreter
(tests/plan_sim.py).  Gates: FFMA kernels 2e-5 relative to max(1, max|ref|); split TF32 / fp16 split 1e-4; max pooling
and copies bit-exact.  Every conv asserts the engine it ran on, so a case cannot pass through a silent fallback, and an
engine request the op cannot take must be refused when the program is created.

The errors quoted in the docstrings were measured on an H100 80GB HBM3 at 700 W; the whole module runs in about 50 s
there."""
import numpy as np
import pytest
import torch

import op_cases as oc
from mvector import _lib as L

pytestmark = pytest.mark.gpu


def _rel(got, ref, floor=1.0):
    return float(np.abs(got.astype(np.float64) - ref).max() / max(floor, np.abs(ref).max()))


def _run(case):
    b = oc.build(case)
    got, ops = oc.run_gpu(b)
    oc.assert_engines(b, ops)
    return b, got, oc.sim(b)


@pytest.mark.parametrize('name', list(oc.TC_CASES))
def test_conv_schedule_and_tails(name):
    """Tensor-core engines (and the FFMA reference on the reflect / window / add / prologue cases) on multi-tile
    schedules, M / N / K tails, chunk remainders, fp16-split epilogues and the add / BN-ReLU prologue gathers.  Measured
    max-rel error: split TF32 <= 3.2e-6 on the plain source (largest: K = 1600 chunked by 512), <= 1.9e-6 with the add,
    <= 7.9e-6 with the prologue (CAM++'s transit, K = 1024); fp16 split <= 1.8e-6; FFMA <= 1.2e-6."""
    case = oc.TC_CASES[name]
    _, got, ref = _run(case)
    err = _rel(got, ref)
    print(f'{name}: max-rel err {err:.2e}')
    assert err <= (2e-5 if case['engine'] == 'ffma' else 1e-4), err


@pytest.mark.parametrize('name', list(oc.ENGINE_CASES))
def test_conv_engines_on_backbone_geometries(name):
    """The backbones' conv geometries on exact fp32 FFMA, split TF32 and (N >= 128) the fp16 split, and the engine AUTO
    resolves to where a tensor-core engine cannot take the op (FFMA for a prologue with a second source, split TF32 on
    the raw program input), gated by the engine that ran.  Measured max-rel error: FFMA <= 7.5e-6; split TF32 <= 3.7e-6
    at K <= 512 and up to 4.1e-5 at K = 1536, the longest unchunked accumulation -- the tensor core's fp32 accumulator
    truncates on every accumulate, a bias that does not average out, still 10-100x below single-pass TF32's ~1e-3;
    fp16 split <= 2.2e-5 (K = 1536)."""
    b, got, ref = _run(oc.ENGINE_CASES[name])
    err = _rel(got, ref)
    print(f'{name}: max-rel err {err:.2e}')
    assert err <= (2e-5 if b.expect[b.main] == L.ENGINE_FFMA else 1e-4), err


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
    _, got, ref = _run(oc.FFMA_CASES[name])
    err = _rel(got, ref)
    print(f'{name}: max-rel err {err:.2e}')
    assert err <= 2e-5, err


EXACT = {'pool_max_k3s1', 'pool_max_k3s2_negative', 'pool_max_fout1_negative', 'ew_copy_window', 'pad_copy_c201',
         'pad_copy_c257'}


@pytest.mark.parametrize('name', list(oc.GLUE_CASES))
def test_glue_kernels(name):
    """pool2d, ew (GATE_RES / AFF / COPY), pad copy, colstats and ASP.  Max pooling and the copies are bit-exact
    (the pad columns exactly +0); the rest within 2e-5 of max(1, max|ref|), measured <= 4.6e-7.  The near-constant
    colstats columns (mean 1e3, spread 1e-3) also check the spread column on its own: the fp32 mean carries an error of
    about one input ulp, which the centred sum of squares sees as a relative variance error of up to ~1e-2 (measured
    7.2e-3 for the std at R = 800, 1.1e-2 for the variance at R = 1201; a one-pass E[x^2] - E[x]^2 is off by 1e5 and
    more)."""
    case = oc.GLUE_CASES[name]
    b, got, ref = _run(case)
    if name in EXACT:
        assert np.array_equal(got, ref)
        if case.get('mode') == 'PAD_COPY':
            c0 = case.get('out_coff', 0) + case['C']
            pad = got[:, c0:c0 + case['Cout'] - case['C']]
            assert not pad.view(np.uint32).any()                 # +0.0 bits, not just == 0
        return
    err = _rel(got, ref)
    print(f'{name}: max-rel err {err:.2e}')
    assert err <= 2e-5, err
    if case.get('fill', ('normal',))[1:] == (1e-3, 1e3):
        C = case['C']
        spread = np.abs(got[:, C:] - ref[:, C:]) / ref[:, C:]
        print(f'{name}: spread column max-rel err {spread.max():.2e}')
        assert spread.max() <= 5e-2, spread.max()


SCALED = {**oc.AMAX_CASES, **oc.TC16_RANGE_CASES}


@pytest.mark.parametrize('name', list(SCALED))
def test_amax_writer_feeds_tc16(name):
    """Every kernel that writes a TC16 source reports max|y| into the source's amax slot: the consumer (1x1 TC16 conv)
    must stay finite and fp32-grade at input scales 1e-30 ... 1e30 (inputs and writer biases both scaled), and so must
    a 512 x 512 GEMM over 8 x 298 rows (the gemm_512 cases).  A writer that reports too small a maximum gives the
    consumer too large a scale, and its fp16 hi terms overflow at any magnitude; a writer that reports nothing leaves
    the slot at 0, which means scale 1: overflow at the large scales, flush to zero at the small ones.  (Too large a
    maximum -- an over-reporting writer, a stale slot -- flushes small tensors to zero; see the graph-replay test.)
    Measured max-rel error <= 1.7e-6 (2.3e-6 on the 512 x 512 GEMM)."""
    case = SCALED[name]
    b, got, ref = _run(case)
    assert b.pb.ops[b.consumer].amax_in > 0
    assert np.isfinite(got).all()
    err = _rel(got, ref, floor=0.0)
    print(f'{name}: max-rel err {err:.2e}')
    assert err <= 2e-5, err


@pytest.mark.parametrize('order', list(oc.SHARED_SLOT_CASES))
def test_amax_slot_shared_by_column_windows(order):
    """Two ops write the two column windows of one allocation at scales 1e6 and 1; the TC16 consumer reads all of it.
    Both writers max into one slot, whichever writes last."""
    b, got, ref = _run(oc.SHARED_SLOT_CASES[order])
    assert np.isfinite(got).all()
    err = _rel(got, ref, floor=0.0)
    assert err <= 2e-5, err


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
    assert _rel(outs[0], oc.sim(big), floor=0.0) <= 2e-5
    ref = oc.sim(small)
    assert np.isfinite(outs[1]).all() and np.isfinite(outs[2]).all()
    assert _rel(outs[1], ref, floor=0.0) <= 2e-5
    assert np.array_equal(outs[1].view(np.uint32), outs[2].view(np.uint32))
