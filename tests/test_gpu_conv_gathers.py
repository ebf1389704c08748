"""GPU tests of the tensor-core conv's add (conv_tc_kernel<1, ...>) and BN-ReLU prologue (conv_tc_kernel<2, ...>)
gathers, and of the engine mirror the CPU coverage tests rely on.

* Every add / prologue case of tests/op_cases.py (GATHER_CASES, on split TF32 and FFMA) against its MODE 0 twin: the
  same op reading the operand its gather computes, materialised on the host.  The two programs share weights, geometry,
  tile / chunk schedule and epilogue, so their outputs are compared for equality, not within a tolerance: a row,
  channel, slot or padding mix-up in the gather shows however small it is.  (The fp64 error of the same cases is
  test_gpu_op_edges.py::test_conv_schedule_and_tails.)
* op_cases.engine_of against the engines vp_program_create resolves, op by op, for the four bench.py configurations.

Measured on an H100 80GB HBM3 (700 W): every twin comparison bit-exact; the module runs in about 30 s there."""
import numpy as np
import pytest
import torch

import op_cases as oc
from mvector import _lib as L

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', list(oc.GATHER_CASES))
def test_gather_equals_plain_gather_of_its_operand(name):
    case = oc.GATHER_CASES[name]
    b, t = oc.build(case), oc.build(oc.twin(case))
    o, ot = b.pb.ops[b.main], t.pb.ops[t.main]
    assert ot.pre_s < 0 and ot.src2_mode == L.SRC2_NONE and ot.w == o.w and ot.w_tc == o.w_tc
    np.testing.assert_array_equal(t.blob, b.blob)
    got, ops = oc.run_gpu(b)
    want, ops_t = oc.run_gpu(t)
    oc.assert_engines(b, ops)
    oc.assert_engines(t, ops_t)
    eng = ops[b.main]['engine']
    assert ops_t[t.main]['engine'] == eng
    kern, kern_t = oc.kernel_of(o, eng), oc.kernel_of(ot, eng)
    assert kern == case['kernel'] and kern_t == kern.replace(',add', '').replace(',pre', '')
    if eng == L.ENGINE_TC:
        assert oc.tc_schedule(ot, eng) == oc.tc_schedule(o, eng)
    assert np.isfinite(got).all() and np.isfinite(want).all()          # every element stored (NaN-poisoned output)
    bad = got != want                                                  # +0 == -0: the sign of a zero may differ
    assert not bad.any(), f'{int(bad.sum())} elements differ, first at {np.argwhere(bad)[0]}'


@pytest.mark.parametrize('cfg', sorted(oc.BENCH_T))
def test_engine_mirror_matches_program(cfg):
    """Each bench.py configuration lowered at its bench batch and T (the largest workspace, c5's, is 15 GB); the Program
    resolves every op's engine exactly as op_cases.engine_of predicts, and the gather families the coverage tests
    attribute to the model are among the kernels it runs.  Nothing is launched."""
    from mvector.engine import Engine, Program
    model, c = oc.bench_model(cfg)
    pb = model.lower(c['per_gpu'], oc.BENCH_T[cfg])
    eng = Engine()
    try:
        eng.load_weights(model._blob)
        prog = Program(eng, pb)
        got = oc.program_engines(prog)
        prog.close()
    finally:
        eng.close()
    want = [oc.engine_of(o) for o in pb.ops]
    assert got == want, [(i, g, w) for i, (g, w) in enumerate(zip(got, want)) if g != w]
    kernels = {oc.kernel_of(o, e) for o, e in zip(pb.ops, got) if o.kind == L.OP_CONV}
    family = {'c2': 'conv_tc<tf32,add>', 'c3': 'conv_tc<tf32,pre>', 'c5': 'conv_tc<tf32,add>'}.get(cfg)
    assert family is None or family in kernels, kernels
