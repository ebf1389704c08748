"""Op-level GPU tests of the two conv engines (exact fp32 FFMA, wgmma split-TF32) and of the pooling kernels against the
fp64 numpy interpreter (tests/plan_sim.py), over the conv geometries the five backbones use and the input sizes on both
sides of each pooling kernel choice."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _run_case(case, engine_id):
    from mvector import _lib as L
    from mvector.engine import Engine, PlanBuilder, Program, View, WeightArena
    from plan_sim import Sim
    rng = np.random.default_rng(case['seed'])
    B, Tin, Fin, Cin = case['B'], case['Tin'], case.get('Fin', 1), case['Cin']
    Tout, Fout, N = case['Tout'], case.get('Fout', 1), case['N']
    KT, KF = case.get('KT', 1), case.get('KF', 1)
    Cin2 = case.get('Cin2', 0)
    src2_mode = case.get('src2_mode', L.SRC2_NONE)
    cin_tot = Cin + (Cin2 if src2_mode == L.SRC2_CONCAT else 0)
    K = KT * KF * cin_tot
    rows_in, rows_out = B * Tin * Fin, B * Tout * Fout
    n_seg = case.get('n_seg', 1)
    # one wide input matrix: [x | x2 | res(out rows) | gate/ubias rows]
    c_x2 = Cin
    c_res = c_x2 + (Cin2 if src2_mode == L.SRC2_CONCAT else (Cin if src2_mode == L.SRC2_ADD else 0))
    c_gu = c_res + (N if case.get('res') else 0)
    c_sum = c_gu + (2 * N if (case.get('gate') or case.get('ubias')) else 0)
    width = c_sum + (N if case.get('sum') else 0)
    width = (width + 3) // 4 * 4
    rows = max(rows_in, rows_out, B * n_seg)
    X = (rng.standard_normal((rows, width)) * case.get('scale', 1.0)).astype(np.float32)
    arena = WeightArena()
    W = rng.standard_normal((N, K)) / np.sqrt(K)
    w = arena.add_conv('w', W)
    bias = arena.add('b', rng.standard_normal(N) * 0.1) if case.get('bias') else -1
    post = (arena.add('ps', rng.uniform(0.5, 1.5, N)), arena.add('ph', rng.standard_normal(N) * 0.2)) if case.get('post') else None
    pre = (arena.add('qs', rng.uniform(0.5, 1.5, cin_tot)), arena.add('qh', rng.standard_normal(cin_tot) * 0.2)) if case.get('pre') else None
    pb = PlanBuilder(B, engine_id)
    pb.in_floats = rows * width
    inp = View(L.BUF_INPUT, width, 0, width)
    src = inp.cols(0, Cin)
    if engine_id == L.ENGINE_TC16:
        # the fp16 split scales by the source tensor's tracked maximum: the source must be a workspace tensor written by
        # a program op (here: a copy of the input columns), as it always is inside a backbone
        src = pb.alloc(rows_in, Cin)
        pb.ew(L.EW_COPY, inp.cols(0, Cin), src, Tin * Fin)
    src2 = None
    if src2_mode == L.SRC2_ADD:
        src2 = inp.cols(c_x2, Cin)
    elif src2_mode == L.SRC2_CONCAT:
        src2 = inp.cols(c_x2, Cin2)
    res = inp.cols(c_res, N) if case.get('res') else None
    gate = ubias = None
    if case.get('gate'):
        gate = pb.alloc(B * n_seg, N)
        pb.ew(L.EW_COPY, inp.cols(c_gu, N), gate, 1).B = B * n_seg
    if case.get('ubias'):
        ubias = pb.alloc(B * n_seg, N)
        pb.ew(L.EW_COPY, inp.cols(c_gu + N, N), ubias, 1).B = B * n_seg
    n_out = 2 * N if case.get('sum') else N
    out_full = pb.output_view(n_out, rows_out)
    out = out_full.cols(0, N)
    acc = None
    if case.get('sum'):                    # accumulate-into view: prefilled, then acc += conv output (Res2 chains)
        acc = pb.alloc(rows_out, N)
        pb.ew(L.EW_COPY, inp.cols(c_sum, N), acc, Tout * Fout)
    pb.conv(src, out, w, K, Tin, Tout, Fin=Fin, Fout=Fout, KT=KT, KF=KF, sT=case.get('sT', 1), sF=case.get('sF', 1),
            dT=case.get('dT', 1), dF=1, padT=case.get('padT', 0), padF=case.get('padF', 0),
            pad_mode=case.get('pad_mode', L.PAD_ZERO), bias=bias, pre=pre, pre_relu=bool(case.get('pre')), post=post,
            act=case.get('act', L.ACT_NONE), act2=case.get('act2', L.ACT_NONE), res=res, gate=gate, ubias=ubias,
            seg_len=case.get('seg_len'), n_seg=n_seg, src2=src2, src2_mode=src2_mode, sum_into=acc)
    if acc is not None:
        pb.ew(L.EW_COPY, acc, out_full.cols(N, N), Tout * Fout)
    eng = Engine()
    blob = arena.blob()
    eng.load_weights(blob)
    prog = Program(eng, pb)
    y = torch.empty(rows_out, n_out, device='cuda')
    prog.run(torch.from_numpy(X).cuda().contiguous(), y)
    torch.cuda.synchronize()
    ref = Sim(pb, blob, X).run().reshape(rows_out, n_out)
    got = y.cpu().numpy()
    eng.close()
    return got, ref


L_ = None
CASES = dict(
    gemm_512=dict(seed=1, B=8, Tin=298, Tout=298, Cin=512, N=512, bias=True, act=1, post=True),
    gemm_n1536_k128=dict(seed=2, B=5, Tin=298, Tout=298, Cin=128, N=1536, bias=True),
    gemm_k1536_n128_ubias_tanh=dict(seed=3, B=6, Tin=211, Tout=211, Cin=1536, N=128, ubias=True, act=1, post=True, act2=4),
    res2_k3_dil2_reflect_add=dict(seed=4, B=9, Tin=298, Tout=298, Cin=64, N=64, KT=3, dT=2, padT=2, pad_mode=1, bias=True,
                                  act=1, post=True, src2_mode=1),
    stem_k5_reflect=dict(seed=5, B=7, Tin=298, Tout=298, Cin=80, N=512, KT=5, padT=2, pad_mode=1, bias=True, act=1, post=True),
    tdnn_valid_k3_d3=dict(seed=6, B=4, Tin=300, Tout=294, Cin=512, N=512, KT=3, dT=3, bias=True, act=1, post=True),
    conv2d_3x3_s2=dict(seed=7, B=3, Tin=61, Fin=40, Tout=31, Fout=20, Cin=32, N=48, KT=3, KF=3, sT=2, sF=2, padT=1, padF=1,
                       bias=True, act=2),
    conv2d_3x3_res_relu=dict(seed=8, B=2, Tin=50, Fin=20, Tout=50, Fout=20, Cin=32, N=32, KT=3, KF=3, padT=1, padF=1, bias=True,
                             res=True, act2=1),
    concat_1x1_silu=dict(seed=9, B=2, Tin=40, Fin=30, Tout=40, Fout=30, Cin=16, Cin2=16, N=16, bias=True, act=5, src2_mode=2),
    cam_pre_bn_relu=dict(seed=10, B=9, Tin=149, Tout=149, Cin=160, N=128, pre=True, bias=True, act=1),
    cam_local_gate_seg=dict(seed=11, B=6, Tin=249, Tout=249, Cin=128, N=32, KT=3, dT=2, padT=2, gate=True, seg_len=100, n_seg=3),
    k5_stride2_zero=dict(seed=12, B=8, Tin=298, Tout=149, Cin=320, N=128, KT=5, sT=2, padT=2, bias=True, act=1),
    n_tail_192=dict(seed=13, B=3, Tin=400, Tout=400, Cin=96, N=192, bias=True),
    long_k_chunked_9216=dict(seed=15, B=6, Tin=40, Fin=20, Tout=20, Fout=10, Cin=1024, N=256, KT=3, KF=3, sT=2, sF=2, padT=1, padF=1),
    long_k_chunked_4096_n128=dict(seed=16, B=7, Tin=151, Tout=151, Cin=4096, N=128, ubias=True, act=1, post=True, act2=4),
    res2_k3_dil3_reflect_sum=dict(seed=17, B=9, Tin=298, Tout=298, Cin=64, N=64, KT=3, dT=3, padT=3, pad_mode=1, bias=True,
                                  act=1, post=True, sum=True),
    conv2d_3x3_sum_hardtanh=dict(seed=18, B=2, Tin=50, Fin=20, Tout=50, Fout=20, Cin=16, N=16, KT=3, KF=3, padT=1, padF=1,
                                 bias=True, act=2, sum=True),
    k_tail_72=dict(seed=14, B=11, Tin=100, Tout=100, Cin=24, N=24, KT=3, padT=1, bias=True, act=2),
)


@pytest.mark.parametrize('name', list(CASES))
def test_conv_ffma_engine_exact(name):
    from mvector import _lib as L
    got, ref = _run_case(CASES[name], L.ENGINE_FFMA)
    assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize('name', list(CASES))
def test_conv_tc_engine_split_tf32(name):
    """wgmma split-TF32 engine: fp32-grade (error << single-pass TF32's ~1e-3)."""
    from mvector import _lib as L
    got, ref = _run_case(CASES[name], L.ENGINE_TC)
    err = np.abs(got - ref).max() / max(1.0, np.abs(ref).max())
    # measured: ~1e-6 at K <= 512, growing ~linearly with K (4.8e-5 at K=1536): the tensor core's fp32 accumulator
    # truncates (RZ) on every accumulate, a bias that does not average out; still 10-100x below single-pass TF32.
    assert err <= 1e-4, err
    print(f'{name}: max-rel err {err:.2e}')


TC16_CASES = ['gemm_512', 'gemm_n1536_k128', 'gemm_k1536_n128_ubias_tanh', 'stem_k5_reflect', 'tdnn_valid_k3_d3',
              'k5_stride2_zero', 'n_tail_192', 'long_k_chunked_9216', 'long_k_chunked_4096_n128']


@pytest.mark.parametrize('name', TC16_CASES)
def test_conv_tc16_engine_fp16_split(name):
    """wgmma two-term FP16 split (VP_ENGINE_TC16) with the dynamic power-of-two activation scale: fp32-grade."""
    from mvector import _lib as L
    got, ref = _run_case(CASES[name], L.ENGINE_TC16)
    err = np.abs(got - ref).max() / max(1.0, np.abs(ref).max())
    assert err <= 1e-4, err
    print(f'{name}: max-rel err {err:.2e}')


@pytest.mark.parametrize('scale', [1e-30, 1e-8, 1e-3, 1e4, 1e9, 1e30])
def test_conv_tc16_is_range_safe(scale):
    """Un-normalised activations: the fp16 split must neither overflow (|x| > 65504) nor lose small tensors to fp16
    subnormals -- the scale comes from the tensor's tracked maximum, so the relative error does not depend on magnitude."""
    from mvector import _lib as L
    case = dict(CASES['gemm_512'], post=False, bias=False, act=0, scale=scale, seed=31)
    got, ref = _run_case(case, L.ENGINE_TC16)
    assert np.isfinite(got).all()
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err <= 2e-5, (scale, err)


def test_conv_tc16_refused_without_tracked_source():
    """A CONV reading the raw program input has no amax slot: an explicit TC16 request is refused, AUTO picks split TF32."""
    from mvector import _lib as L
    from mvector.engine import Engine, PlanBuilder, Program, View, WeightArena
    rng = np.random.default_rng(0)
    arena = WeightArena()
    w = arena.add_conv('w', rng.standard_normal((256, 256)) / 16)
    for pref, expect in ((L.ENGINE_TC16, None), (L.ENGINE_AUTO, L.ENGINE_TC)):
        pb = PlanBuilder(8, pref)
        pb.in_floats = 8 * 200 * 256
        pb.conv(View(L.BUF_INPUT, 256, 0, 256), pb.output_view(256, 8 * 200), w, 256, 200, 200)
        eng = Engine()
        eng.load_weights(arena.blob())
        if expect is None:
            with pytest.raises(L.VpError):
                Program(eng, pb)
        else:
            prog = Program(eng, pb)
            y = torch.empty(8 * 200, 256, device='cuda')
            ops = prog.run_profiled(torch.randn(8 * 200 * 256, device='cuda'), y)
            assert ops[0]['engine'] == expect
        eng.close()


PRE_SRC2 = dict(
    pre_concat_1x1=dict(seed=21, B=9, Tin=149, Tout=149, Cin=96, Cin2=64, N=128, pre=True, bias=True, act=1, src2_mode=2),
    pre_add_k3=dict(seed=22, B=9, Tin=149, Tout=149, Cin=64, N=64, KT=3, padT=1, pre=True, bias=True, act=1, src2_mode=1),
)


@pytest.mark.parametrize('name', list(PRE_SRC2))
def test_prologue_with_second_source_engine_ab(name):
    """ADVICE r1: a BN-ReLU prologue combined with a second source (add / concat).  The tensor-core gather (MODE 2) reads one
    source, so ENGINE_AUTO must route the op to the FFMA engine (exact vs the interpreter) and an explicit ENGINE_TC
    request must be refused loudly -- never a silently different result."""
    from mvector import _lib as L
    got, ref = _run_case(PRE_SRC2[name], L.ENGINE_AUTO)
    assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())
    got, ref = _run_case(PRE_SRC2[name], L.ENGINE_FFMA)
    assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())
    with pytest.raises(L.VpError):
        _run_case(PRE_SRC2[name], L.ENGINE_TC)


def _run_pool(case):
    """One ASP_POOL (mean_only: SAP) or COLSTATS op on columns [coff, coff + C) (x) and [coff + C, coff + 2 C) (logits)
    of a random input."""
    from mvector import _lib as L
    from mvector.engine import Engine, PlanBuilder, Program, View, WeightArena
    from plan_sim import Sim
    rng = np.random.default_rng(case['seed'])
    B, R, C, coff = case['B'], case['R'], case['C'], case.get('coff', 0)
    width = (coff + 2 * C + 3) // 4 * 4
    X = (rng.standard_normal((B * R, width)) * 2).astype(np.float32)
    arena = WeightArena()
    arena.add('unused', np.zeros(4))
    pb = PlanBuilder(B, L.ENGINE_AUTO)
    pb.in_floats = B * R * width
    inp = View(L.BUF_INPUT, width, 0, width)
    x = inp.cols(coff, C)
    if 'stats' in case:
        mode = getattr(L, 'STATS_' + case['stats'])
        seg_len = case.get('seg_len')
        n_seg = -(-R // seg_len) if seg_len else 1
        n_rows = B * n_seg
        n_cols = C if mode in (L.STATS_MEAN, L.STATS_SEG_CONTEXT) else 2 * C
        pb.colstats(x, pb.output_view(n_cols, n_rows), R, mode, eps=1e-5, seg_len=seg_len, n_seg=n_seg)
    else:
        n_rows, n_cols = B, C if case['mean_only'] else 2 * C
        pb.asp_pool(x, inp.cols(coff + C, C), pb.output_view(n_cols, n_rows), R, eps=1e-12, mean_only=case['mean_only'])
    eng = Engine()
    blob = arena.blob()
    eng.load_weights(blob)
    y = torch.empty(n_rows, n_cols, device='cuda')
    Program(eng, pb).run(torch.from_numpy(X).cuda().contiguous(), y)
    torch.cuda.synchronize()
    ref = Sim(pb, blob, X).run().reshape(n_rows, n_cols)
    got = y.cpu().numpy()
    eng.close()
    return got, ref


POOL_CASES = {}
# ASP / mean-only SAP: the [T, 32] strips of x and logits are staged in shared memory up to T = 800 (T * 256 B <= 200 KB)
for _T in (400, 401, 800, 801):
    POOL_CASES[f'asp_T{_T}'] = dict(mean_only=False, B=3, R=_T, C=72, seed=_T)
    POOL_CASES[f'sap_mean_T{_T}'] = dict(mean_only=True, B=3, R=_T, C=72, seed=_T + 1)
# colstats: the [R, 32] strip is staged in shared memory up to R = 800 rows (R * 128 B <= 100 KB)
for _i, _stats in enumerate(('MEAN', 'MEAN_STD_CLAMP', 'MEAN_STD_UNBIASED', 'MEAN_STD_TSTP', 'MEAN_VAR_UNBIASED')):
    for _R in (800, 801):
        POOL_CASES[f'colstats_{_stats.lower()}_R{_R}'] = dict(stats=_stats, B=3, R=_R, C=72, seed=_R + _i)
# segment context: the segment sums are parked in shared memory up to 64 segments, two sweeps above
for _n in (64, 65):
    POOL_CASES[f'seg_context_{_n}'] = dict(stats='SEG_CONTEXT', B=3, R=10 * _n - 5, C=72, seg_len=10, seed=_n)
# views that start one column into their matrix: no 16-byte staging, the global-memory kernels run
POOL_CASES['asp_unaligned_coff'] = dict(mean_only=False, B=3, R=298, C=72, coff=1, seed=7)
POOL_CASES['colstats_unaligned_coff'] = dict(stats='MEAN_STD_CLAMP', B=3, R=298, C=72, coff=1, seed=8)


@pytest.mark.parametrize('name', list(POOL_CASES))
def test_pool_kernels_match_interpreter(name):
    got, ref = _run_pool(POOL_CASES[name])
    assert np.abs(got - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())
