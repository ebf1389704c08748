"""GPU tests of the fp16 split's wide path (conv_tc.cu conv_tc16_wide_kernel): 128 x 256 tiles with TMA-loaded fp32
activations split in the consumer warps, taken by pointwise, stride-1, unpadded, unchunked convs with one plain source,
N % 256 == 0 and N >= 1024 (tc16_wide_ok).

- Its first 128 columns equal the 128-wide kernel's output bit for bit: same operands, same K order (A_lo B_hi,
  A_hi B_lo, A_hi B_hi per K16 step into one accumulator), same epilogue.
- Its edges (M and K tails, column windows of a wider input and output, the fused epilogue, 32 and 152 tiles per launch,
  activations at 1e-30 and 1e+30) match the fp64 interpreter (tests/plan_sim.py) at the engine's 1e-4 gate.
- Convs outside the predicate still launch the 128-wide kernel, and pointwise ones inside it launch the wide one:
  checked by kernel name in a torch.profiler trace."""
import numpy as np
import pytest
import torch

import op_cases as oc
from mvector import _lib as L
from mvector.engine import PlanBuilder, View, WeightArena

pytestmark = pytest.mark.gpu

WIDE = 'conv_tc16_wide_kernel'
NARROW = 'conv_tc_kernel<0, true'


def _rel(got, ref, floor=1.0):
    return float(np.abs(got.astype(np.float64) - ref).max() / max(floor, np.abs(ref).max()))


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
    assert _rel(got, oc.sim(b)) <= 1e-4


def _case(seed, **c):
    return dict(op='conv', engine='tc16', kernel='conv_tc<f16>', seed=seed, **c)


EDGE_CASES = {
    'm_tail': _case(201, B=3, Tin=683, Cin=512, N=1024, bias=True, act=L.ACT_RELU),           # M = 2049
    'k_tail': _case(202, B=2, Tin=700, Cin=72, N=1024, bias=True),                             # K = 72 = 64 + 8
    'k_tail_136': _case(203, B=2, Tin=700, Cin=136, N=1280, bias=True, act=L.ACT_RELU),
    'in_window': _case(204, B=4, Tin=300, Cin=512, in_coff=1024, N=1536, bias=True),          # cat slice, in_ld 1536
    'out_window': _case(205, B=4, Tin=300, Cin=128, N=1024, out_coff=516, bias=True, act=L.ACT_RELU),
    'relu_bn_res': _case(206, B=4, Tin=300, Cin=512, N=1536, bias=True, act=L.ACT_RELU, post=True, res=True),
    'res_act2_tail': _case(207, B=3, Tin=683, Cin=128, N=1024, bias=True, res=True, act2=L.ACT_RELU),
    'tiles_4': _case(208, B=1, Tin=1024, Cin=256, N=1024, bias=True),                          # 8 x 4 tiles on 32 CTAs
    'tiles_152': _case(209, B=8, Tin=300, Cin=128, N=2048, bias=True, act=L.ACT_RELU),         # 19 x 8 on 132 CTAs
    'general_epilogue': _case(210, B=4, Tin=300, Cin=128, N=1024, bias=True, ubias=True, act=L.ACT_SILU),
    'scale_1e-30': _case(211, B=4, Tin=300, Cin=512, N=1024, bias=True, bias_scale=1e-30, scale=1e-30),
    'scale_1e+30': _case(212, B=4, Tin=300, Cin=512, N=1024, bias=True, bias_scale=1e30, scale=1e30),
}


@pytest.mark.parametrize('name', list(EDGE_CASES))
def test_wide_path_edges(name):
    """Every edge runs on the wide kernel and matches the fp64 interpreter at the fp16 split's 1e-4 gate, relative to
    max|ref| (floor 1, except the range cases: relative to max|ref| alone)."""
    case = EDGE_CASES[name]
    b = oc.build(case)
    got, names = _kernels(b)
    assert any(WIDE in n for n in names) and not any(NARROW in n for n in names), names
    assert np.isfinite(got).all()
    err = _rel(got, oc.sim(b), floor=0.0 if 'scale' in case else 1.0)
    print(f'{name}: max-rel err {err:.2e}')
    assert err <= 1e-4, err


ROUTING_CASES = {
    'n512': _case(305, B=4, Tin=300, Cin=512, N=512, bias=True, act=L.ACT_RELU, post=True),
    'n1152': _case(301, B=4, Tin=300, Cin=512, N=1152, bias=True, act=L.ACT_RELU),
    'chunked_k2048': _case(302, B=4, Tin=300, Cin=2048, N=1024, bias=True),                    # tc_kc > 0
    'k3_taps': _case(303, B=4, Tin=300, Cin=128, N=512, KT=3, padT=1, bias=True, act=L.ACT_RELU),
    'concat': _case(304, B=4, Tin=300, Cin=128, Cin2=128, src2_mode=L.SRC2_CONCAT, N=1024, bias=True),
}


@pytest.mark.parametrize('name', list(ROUTING_CASES))
def test_outside_the_predicate_runs_128_wide(name):
    """N < 1024, N % 256 != 0, chunked accumulation, taps, a second source: the 128-wide kernel, at its usual
    accuracy."""
    b = oc.build(ROUTING_CASES[name])
    got, names = _kernels(b)
    assert any(NARROW in n for n in names) and not any(WIDE in n for n in names), names
    err = _rel(got, oc.sim(b))
    print(f'{name}: max-rel err {err:.2e}')
    assert err <= 1e-4, err
