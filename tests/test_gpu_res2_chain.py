"""The fused Res2Net chain (conv_tc.cu res2_chain_kernel, picked in vp_program_create by res2_chain_len): a chain of
split-TF32 k3 reflect convs y_j = conv_j(t1_j + y_{j-1}) run as one launch must equal the same ops run one op per
program (a single op never fuses) bit for bit, through every launch path, and must leave the columns around its
windows untouched."""
import numpy as np
import pytest
import torch

from mvector import _lib as L
from mvector.engine import Engine, PlanBuilder, Program, View, WeightArena

from op_cases import assert_bit_identical

pytestmark = pytest.mark.gpu


def t_limit(w, d):
    """Largest T the fused kernel takes (conv_tc.cu res2_chain_supported: two weight stages and the hi / lo planes of
    T + 2d rows, rounded to 4 mod 8, within 226 KB of shared memory; at most 384 frames)."""
    t = 384
    while t > 0:
        rows = (t + 2 * d + 3) // 8 * 8 + 4
        if 1024 + 2 * 2 * w * 128 + 2048 + 2 * (w // 4) * rows * 16 + 1024 <= 226 * 1024:
            return t
        t -= 1
    return 0


def _chain(B, T, w, d, n, seed, acts=None, tracked=False, in_pad=12, out_pad=8):
    """-> (per-op PlanBuilders, the whole-chain PlanBuilder, blob, X, out shape).  t1 is the column window
    [in_pad, in_pad + n w) of the input, y the window [out_pad, out_pad + n w) of the output.  acts: each op's
    activation (ReLU throughout by default).  tracked: the whole-chain program writes y into a workspace tensor that an
    FP16-split conv reads as its source, so that the chain ops max |y| into that tensor's amax slot, and copies y out."""
    acts = acts or [L.ACT_RELU] * n
    rng = np.random.default_rng(seed)
    arena = WeightArena()
    K = 3 * w
    ws = [dict(w=arena.add_conv(f'w{j}', rng.standard_normal((w, K)) / np.sqrt(K)),
               b=arena.add(f'b{j}', rng.standard_normal(w) * 0.1),
               s=arena.add(f's{j}', rng.uniform(0.5, 1.5, w)), h=arena.add(f'h{j}', rng.standard_normal(w) * 0.2))
          for j in range(n)]
    wc = arena.add_conv('wc', rng.standard_normal((128, n * w)) / np.sqrt(n * w))
    rows = B * T
    in_w, out_w = in_pad + n * w + 4, out_pad + n * w + 8 + (128 if tracked else 0)
    X = rng.standard_normal((rows, in_w)).astype(np.float32)
    t1 = View(L.BUF_INPUT, in_w, in_pad, n * w)
    y_out = View(L.BUF_OUTPUT, out_w, out_pad, n * w)

    def emit(pb, y, j):
        pb.conv(t1.cols(j * w, w), y.cols(j * w, w), ws[j]['w'], K, T, T, KT=3, dT=d, padT=d, pad_mode=L.PAD_REFLECT,
                bias=ws[j]['b'], act=acts[j], post=(ws[j]['s'], ws[j]['h']),
                src2=y.cols((j - 1) * w, w) if j else None, src2_mode=L.SRC2_ADD if j else L.SRC2_NONE,
                engine=L.ENGINE_TC)

    def builder(js, tracked=False):
        pb = PlanBuilder(B)
        pb.input_view(in_w, rows)
        pb.output_view(out_w, rows)
        y = pb.alloc(rows, n * w) if tracked else y_out
        for j in js:
            emit(pb, y, j)
        if tracked:
            pb.conv(y, View(L.BUF_OUTPUT, out_w, out_pad + n * w + 8, 128), wc, n * w, T, T)
            pb.ew(L.EW_COPY, y, y_out, T)
        return pb

    return [builder([j]) for j in range(n)], builder(range(n), tracked), arena.blob(), X, (rows, out_w)


def _slot(prog, pb, q):
    """amax slot q (1-based) of a Program after its run, as float32 (vp_program_peek reads the slots behind the
    workspace)."""
    import ctypes as C
    buf = torch.zeros(1, dtype=torch.int32, device='cuda')
    off = (max(pb.peak, 256) + 255) // 256 * 256 + 4 * (q - 1)
    assert L.lib().vp_program_peek(prog._p, off, 4, C.c_void_p(buf.data_ptr()), prog.engine.stream_ptr()) == L.VP_OK
    torch.cuda.synchronize()
    return buf.cpu().numpy().view(np.float32)[0]


def _run(B, T, w, d, n, seed=0, acts=None, tracked=False):
    """-> (fused output, per-op output, fused Program launches, profiled records of the fused program, the amax slot of
    y after the fused run or None)"""
    singles, whole, blob, X, shape = _chain(B, T, w, d, n, seed, acts, tracked)
    eng = Engine()
    try:
        eng.load_weights(blob)
        x = torch.from_numpy(X).cuda()
        y = torch.empty(shape, device='cuda')
        y.fill_(float('nan'))
        for pb in singles:                       # one op per program, in order, on one output tensor
            Program(eng, pb).run(x, y)
        torch.cuda.synchronize()
        ref = y.cpu().numpy()
        prog = Program(eng, whole)
        runs, recs = {}, None
        for label, fn in (('eager', prog.run), ('profiled', prog.run_profiled), ('captured', prog.run),
                          ('replayed', prog.run)):
            y.fill_(float('nan'))
            r = fn(x, y)
            if label == 'profiled':
                recs = r
            torch.cuda.synchronize()
            runs[label] = y.cpu().numpy()
        assert_bit_identical(runs)
        q = whole.ops[0].amax_out
        return runs['eager'], ref, prog.launches, recs, (_slot(prog, whole, q) if q > 0 else None)
    finally:
        eng.close()


CASES = [  # (B, T, w, d, n)
    (256, 298, 64, 2, 7), (256, 298, 64, 3, 7), (256, 298, 64, 4, 7),
    (131, 65, 16, 2, 2), (132, 64, 32, 3, 3), (133, 63, 48, 4, 5), (300, 17, 64, 4, 6),
    (1100, 3, 64, 2, 2), (1030, 4, 32, 3, 4),
    (5, 298, 48, 2, 7), (16, t_limit(64, 4), 64, 4, 7), (16, t_limit(16, 2), 16, 2, 3),
]


@pytest.mark.parametrize('B,T,w,d,n', CASES)
def test_fused_equals_per_op(B, T, w, d, n):
    fused, ref, launches, recs, _ = _run(B, T, w, d, n)
    assert_bit_identical(dict(per_op=ref, fused=fused))
    out_pad = 8
    assert np.isnan(fused[:, :out_pad]).all() and np.isnan(fused[:, out_pad + n * w:]).all()
    assert np.isfinite(fused[:, out_pad:out_pad + n * w]).all()
    assert launches == 1, launches                   # the whole chain is one launch
    assert all(r['engine'] == L.ENGINE_TC for r in recs)


@pytest.mark.parametrize('B,T,w,d,n', [(256, 298, 64, 2, 7), (133, 63, 48, 4, 5)])
def test_amax_slot(B, T, w, d, n):
    """With y tracked, the fused chain's amax slot holds max |y| of the per-op outputs exactly."""
    from mvector import engine as E
    if not E.TC_F16:
        pytest.skip('VPB_TC_F16=0: no fp16 consumer, so no amax slot')
    fused, ref, launches, _, slot = _run(B, T, w, d, n, tracked=True)
    out_pad = 8
    win = slice(out_pad, out_pad + n * w)
    assert_bit_identical(dict(per_op=ref[:, win], fused=fused[:, win]))
    assert np.isnan(fused[:, :out_pad]).all() and np.isnan(fused[:, out_pad + n * w:out_pad + n * w + 8]).all()
    assert launches == 1 + 2 + 1, launches           # memset of the slots, the chain, the fp16 conv, the copy
    assert slot is not None and slot.view(np.uint32) == np.abs(ref[:, win]).max().view(np.uint32), (slot, np.abs(ref[:, win]).max())


@pytest.mark.parametrize('acts,launches', [
    ((L.ACT_RELU, L.ACT_RELU, L.ACT_RELU, L.ACT_NONE, L.ACT_NONE), 3),   # the chain ends where the activation changes
    ((L.ACT_NONE, L.ACT_RELU, L.ACT_RELU), 3),                           # op 0 differs: nothing can fuse behind it
    ((L.ACT_NONE,) * 4, 1),
])
def test_activations(acts, launches):
    n = len(acts)
    fused, ref, got, _, _ = _run(40, 298, 64, 3, n, acts=list(acts))
    assert_bit_identical(dict(per_op=ref, fused=fused))
    assert got == launches, got


def test_above_limit_runs_per_op():
    T = t_limit(64, 4) + 1
    fused, ref, launches, _, _ = _run(4, T, 64, 4, 3)
    assert_bit_identical(dict(per_op=ref, fused=fused))
    assert launches == 3, launches


def _kernels(B, T, w, d, n):
    from torch.profiler import ProfilerActivity, profile
    _, whole, blob, X, shape = _chain(B, T, w, d, n, 0)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng = Engine()
        try:
            eng.load_weights(blob)
            prog = Program(eng, whole)
            x, y = torch.from_numpy(X).cuda(), torch.empty(shape, device='cuda')
            prog.run(x, y)
            prog.run_profiled(x, y)
            torch.cuda.synchronize()
        finally:
            eng.close()
    return [e.key for e in prof.key_averages()]


def test_routing_by_limit():
    lim = t_limit(64, 3)
    assert any('res2_chain_kernel' in k for k in _kernels(8, lim, 64, 3, 3))
    above = _kernels(8, lim + 1, 64, 3, 3)
    assert not any('res2_chain_kernel' in k for k in above) and any('conv_tc_kernel' in k for k in above)


def _ecapa():
    from mvector.models import build_model
    from mvector.utils.utils import dict_to_object
    from oracle import models as om
    margs = dict(embd_dim=192, pooling_type='ASP', channels=[512, 512, 512, 512, 1536])
    m = build_model(80, dict_to_object({'model_conf': {'model': 'EcapaTdnn', 'model_args': margs}}))
    m.load_state_dict(om.random_state_dict('EcapaTdnn', 80, seed=0, **margs))
    return m


def test_ecapa_launches():
    """The c2 ECAPA program fuses each SE-Res2 block's seven chain convs: 6 launches fewer per block."""
    m = _ecapa()
    B, T = 256, 298
    ops = m.lower(B, T).finalize().ops
    memset = int(any(o.amax_out > 0 or o.amax_in > 0 for o in ops))
    prog = m.program(B, T)
    assert prog.launches == prog.n_ops + memset - 3 * 6, (prog.n_ops, memset, prog.launches)
    recs = prog.run_profiled(torch.randn(B, T, 80, device='cuda'), torch.empty(B, 192, device='cuda'))
    assert sum(r['kind'] == L.OP_CONV and r['engine'] == L.ENGINE_TC and r['N'] == 64 for r in recs) == 21


class _OneOp:
    """One op of a lowered program, on the program's whole workspace plan: run in order on the handle's shared arena,
    such one-op programs compute what the whole program computes, none of them fusing."""

    def __init__(self, pb, op):
        self.ops, self.peak, self.in_floats, self.out_floats, self.taps = [op], pb.peak, pb.in_floats, pb.out_floats, {}

    def finalize(self):
        return self


_FULL_MODEL = r"""
import sys, numpy as np, torch
sys.path[:0] = ['tests']
import test_gpu_res2_chain as t
from mvector.engine import Program
m = t._ecapa()
B, T = 256, 298
pb = m.lower(B, T).finalize()
assert not any(o.amax_out > 0 or o.amax_in > 0 for o in pb.ops)      # no slots to zero between one-op programs
prog = m.program(B, T)
assert prog.launches == prog.n_ops - 3 * 6
f = torch.randn(B, T, 80, generator=torch.Generator().manual_seed(5)).cuda()
e = torch.empty(B, 192, device='cuda')
prog.run(f, e)
torch.cuda.synchronize()
fused = dict(emb=e.cpu().numpy(), **{k: prog.peek(k).cpu().numpy() for k in prog.taps})
singles = [Program(m.engine, t._OneOp(pb, o)) for o in pb.ops]
e.fill_(float('nan'))
for p in singles:
    p.run(f, e)
torch.cuda.synchronize()
per_op = dict(emb=e.cpu().numpy(), **{k: prog.peek(k).cpu().numpy() for k in prog.taps})
assert len(fused) > 3
for k in fused:
    t.assert_bit_identical({'fused ' + k: fused[k], 'per-op ' + k: per_op[k]})
print('FULL MODEL OK', len(fused))
"""


def test_ecapa_fused_equals_per_op():
    """The c2 ECAPA program (B = 256, T = 298) against the same op list run one op per program on the handle's shared
    arena: embeddings and every block tap bit for bit.  Run without the fp16 images (VPB_TC_F16=0, a fresh process):
    every run of a program zeroes its amax slots, so one-op programs cannot carry a slot from its writers to the fp16
    conv that reads it; the slot itself is checked by test_amax_slot and the fp16 path end to end by the benchmark's
    embeddings."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, VPB_TC_F16='0', PYTHONPATH=os.pathsep.join(p for p in sys.path if p))
    r = subprocess.run([sys.executable, '-c', _FULL_MODEL], cwd=root, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0 and 'FULL MODEL OK' in r.stdout, (r.stdout[-2000:], r.stderr[-3000:])
