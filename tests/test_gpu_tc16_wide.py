"""GPU tests of the fp16 split's wide path (conv_tc.cu conv_tc16_wide_kernel): 128 x 256 tiles with TMA-loaded fp32
activations split in the consumer warps, taken by pointwise, stride-1, unpadded, unchunked convs with one plain source,
N % 256 == 0 and N >= 1024 (tc16_wide_ok).

- Its first 128 columns equal the 128-wide kernel's output bit for bit: same operands, same K order (A_lo B_hi,
  A_hi B_lo, A_hi B_hi per K16 step into one accumulator), same epilogue.
- Its edges (op_cases.TC16_WIDE_CASES: M and K tails, one partial or one full K block, column windows of a wider input
  and output, every epilogue feature, 32, 133, 152 and 252 tiles per launch, activations at 2^-110, 1e-30, 1e+30 and
  2^116) match the fp64 interpreter (tests/plan_sim.py) element by element within the bound of the fp16 split's
  arithmetic (tests/error_bound.py): max |got - ref| / beta <= 1, printed as err/beta beside the old max-rel metric.
- Convs outside the predicate still launch the 128-wide kernel, and pointwise ones inside it launch the wide one:
  checked by kernel name in a torch.profiler trace."""
import numpy as np
import pytest
import torch

import error_bound as eb
import op_cases as oc
from mvector import _lib as L
from mvector.engine import PlanBuilder, View, WeightArena

pytestmark = pytest.mark.gpu

WIDE = 'conv_tc16_wide_kernel'
NARROW = 'conv_tc_kernel<0, true'


_rel = eb.max_rel


def _check(name, b, got, floor=1.0):
    ref, beta = eb.bounded(b)
    r = eb.ratio(got, ref, beta)
    print(f'{name}: err/beta {r:.3f}, max-rel err {_rel(got, ref, floor):.2e}')
    assert r <= 1.0, r


def _pair(K, seed, B=8, T=300, N=1024):
    """One source, two fp16-split convs: N = 1024 with W [1024, K] (wide path) into output columns [0, 1024), and
    N = 128 with W[:128] (128-wide kernel) into [1024, 1152).  W's largest element sits in its first 128 rows, so both
    weight images get the same power-of-two scale; both convs read the same tracked source, so the same activation
    scale."""
    rng = np.random.default_rng(seed)
    rows = B * T
    W = rng.standard_normal((N, K)) / np.sqrt(K)
    W[0, 0] = 2.0 * np.abs(W).max()
    bias = rng.standard_normal(N) * 0.1
    arena = WeightArena()
    arena.add('unused', np.zeros(4))
    pb = PlanBuilder(B, L.ENGINE_AUTO)
    src = pb.alloc(rows, K)
    oc._copy(pb, View(L.BUF_INPUT, K, 0, K), src, rows)
    out = pb.output_view(N + 128, rows)
    pb.conv(src, out.cols(0, N), arena.add_conv('wN', W), K, T, T, bias=arena.add('bN', bias),
            act=L.ACT_RELU, engine=L.ENGINE_TC16)
    pb.conv(src, out.cols(N, 128), arena.add_conv('w128', W[:128]), K, T, T, bias=arena.add('b128', bias[:128]),
            act=L.ACT_RELU, engine=L.ENGINE_TC16)
    pb.in_floats = rows * K
    X = rng.standard_normal((rows, K)).astype(np.float32)
    return oc.Built({}, pb, arena, X, rows, N + 128, 1, {1: L.ENGINE_TC16, 2: L.ENGINE_TC16})


def _kernels(b):
    """Run a built case under torch.profiler -> (output, names of the CUDA kernels it launched)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        got, ops = oc.run_gpu(b)
    oc.assert_engines(b, ops)
    return got, [e.key for e in prof.key_averages()]


@pytest.mark.parametrize('K', [1536, 512, 128])
def test_wide_tile_equals_128_wide_kernel(K):
    """MFA-like (K = 1536), 512-channel and ASP-logits-like (128) operands: the N = 1024 op's first 128 columns are
    bit-identical to the N = 128 op on the same weights, and the two ran on the two different kernels."""
    b = _pair(K, seed=K)
    got, names = _kernels(b)
    assert any(WIDE in n for n in names) and any(NARROW in n for n in names), names
    assert np.isfinite(got).all()
    assert np.array_equal(got[:, :128], got[:, -128:]), np.abs(got[:, :128] - got[:, -128:]).max()
    _check(f'K = {K}', b, got)


WIDE_CASES = {n: c for n, c in oc.TC16_WIDE_CASES.items() if c['kernel'] == 'conv_tc16_wide'}
ROUTING_CASES = {n: c for n, c in oc.TC16_WIDE_CASES.items() if c['kernel'] != 'conv_tc16_wide'}


@pytest.mark.parametrize('name', list(WIDE_CASES))
def test_wide_path_edges(name):
    """Every edge runs on the wide kernel and stays within its per-element bound.  Measured max-rel error <= 2.3e-6
    (2.6e-6 at 1e+-30; 1.7e-7 for the single partial K block of K = 8), relative to max|ref| (floor 1, except the
    range cases: relative to max|ref| alone)."""
    case = WIDE_CASES[name]
    b = oc.build(case)
    got, names = _kernels(b)
    assert any(WIDE in n for n in names) and not any(NARROW in n for n in names), names
    assert np.isfinite(got).all()
    _check(name, b, got, floor=0.0 if 'scale' in case else 1.0)


@pytest.mark.parametrize('name', list(ROUTING_CASES))
def test_outside_the_predicate_runs_128_wide(name):
    """N < 1024, N % 256 != 0, chunked accumulation, taps, a second source: the 128-wide kernel, at its usual
    accuracy."""
    b = oc.build(ROUTING_CASES[name])
    got, names = _kernels(b)
    assert any(NARROW in n for n in names) and not any(WIDE in n for n in names), names
    _check(name, b, got)
