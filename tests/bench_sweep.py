"""Op-by-op sweep of a whole lowered program (tests/test_gpu_bench_programs.py on the GPU, tests/test_bench_programs_cpu.py
on the CPU).  Never imported by the product.

The program is run as its prefixes: prefix i is the finalized plan cut after op i (``prefix``), so it runs the same
kernel instances, amax slots and engines as the full program.  After prefix i the sweep reads op i's outputs and the
operands of op i + 1 from the backend's memory, on the rows ``sample_rows`` picks, and holds each op to its own
rounding: the reference (error_bound.BoundSim.op) starts from the backend's own fp32 operands with bound 0, so an
element above its bound is an error of that op alone, whatever the ops before it did.

The fp16 split of a tensor-core conv scales by the maximum over every window of its source allocation written so far
(PlanBuilder.finalize: one slot per allocation), so the sweep folds max |output| of every writer of a slotted
allocation into a running maximum, over the writer's whole output view, and takes the consumer's design exponent from
that maximum.

A backend runs prefixes and reads views: ``run(pb_prefix)``, ``rows(view, rows)`` (fp32 [len(rows), C]),
``amax(view)`` and ``close()``; ``view`` is an error_bound.views entry.  GpuBackend runs the library; the CPU tests
use an interpreter backend."""
import copy
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np

import error_bound as eb
import op_cases as oc
from mvector import _lib as L

SMS = oc.SMS
EW_STRIDE = 132 * 32 * 256                 # pool.cu launch_ew / launch_pool2d: threads of the capped grid
TC_KERNELS = ('conv_tc', 'conv_tc16_wide')


def prefix(pb, i):
    """The finalized plan cut after op i: ops and their allocation records up to i, the workspace, input and output
    sizes of the full plan, and its amax slots and engines (``_finalized`` stays set, so Program does not re-derive
    them from the shorter op list)."""
    pb.finalize()
    q = copy.copy(pb)
    q.ops, q._meta = pb.ops[:i + 1], pb._meta[:i + 1]
    q._finalized = True
    return q


def is_tc(kernel):
    return kernel.startswith(TC_KERNELS)


def tc_grid(o, eng, kernel):
    """(n_tiles, tiles, grid, BN) of a tensor-core conv's persistent schedule."""
    if kernel == 'conv_tc16_wide':
        sch, bn = oc.wide_schedule(o), oc.WIDE_BN
    else:
        sch = oc.tc_schedule(o, eng)
        bn = sch['bn']
    return sch['n_tiles'], sch['tiles'], min(SMS, sch['tiles']), bn


def locate(o, eng, kernel, m, n):
    """Where output element (m, n) was computed: a dict naming the tile, CTA and ordinal for a tensor-core conv."""
    if not is_tc(kernel):
        return {}
    n_tiles, _, grid, bn = tc_grid(o, eng, kernel)
    g = (m // 128) * n_tiles + n // bn
    return dict(tile=int(g), cta=int(g % grid), ordinal=int(g // grid))


def out_rows(o):
    return eb.views(o)['dst'][4]


def ew_passes(o):
    """[(first float4 index, row width in float4 / elements)] of the grid-stride loop of an ew / pad_copy / pool2d op."""
    per_row = o.Cout if (o.kind == L.OP_EW and o.mode == L.EW_PAD_COPY) else o.Cin // 4
    total = out_rows(o) * per_row
    return -(-total // EW_STRIDE), per_row


def sample_rows(o, eng, kernel, rng, interior=1, spread=64):
    """Output rows of op o to check.

    * tensor-core convs: the M tiles of one tile per CTA index and one tile per ordinal of the persistent schedule
      (tile g runs on CTA g % grid as its (g // grid)-th tile, n-fastest), each at its first, last and ``interior``
      seeded rows, and every row of the first and the last utterance;
    * colstats / asp / linear_small_m: every row;
    * everything else: first and last rows, the rows on both sides of every grid-stride wrap and ``spread`` seeded
      rows."""
    M = out_rows(o)
    if o.kind in (L.OP_COLSTATS, L.OP_ASP_POOL) or kernel == 'linear_small_m':
        return np.arange(M)
    if is_tc(kernel):
        n_tiles, tiles, grid, _ = tc_grid(o, eng, kernel)
        gs = set(range(grid))
        for j in range(-(-tiles // grid)):
            lo = j * grid
            gs.add(lo + int(rng.integers(min(grid, tiles - lo))))
        rows = []
        for mt in sorted({g // n_tiles for g in gs}):
            m0, m1 = mt * 128, min(M, mt * 128 + 128) - 1
            rows += [m0, m1] + rng.integers(m0, m1 + 1, interior).tolist()
        rpu = o.Tout * o.Fout
        rows = np.concatenate([rows, np.arange(rpu), np.arange(M - rpu, M)])
        return np.unique(rows)
    rows = [0, M - 1] + rng.integers(0, M, spread).tolist()
    if o.kind in (L.OP_EW, L.OP_POOL2D):
        passes, per_row = ew_passes(o)
        for k in range(1, passes):
            r = k * EW_STRIDE // per_row
            rows += [r - 1, r]
    return np.unique(np.clip(rows, 0, M - 1))


def tc_coverage(o, eng, kernel, rows):
    """(CTA indices, ordinals) of the tiles whose rows include ``rows`` (every N tile of a sampled M tile is checked)."""
    n_tiles, tiles, grid, _ = tc_grid(o, eng, kernel)
    g = (np.unique(rows // 128)[:, None] * n_tiles + np.arange(n_tiles)[None, :]).reshape(-1)
    g = g[g < tiles]
    return set((g % grid).tolist()), set((g // grid).tolist())


def ew_coverage(o, rows):
    """Grid-stride passes of an ew / pool2d op that ``rows`` reach."""
    _, per_row = ew_passes(o)
    first, last = rows * per_row // EW_STRIDE, ((rows + 1) * per_row - 1) // EW_STRIDE
    return set(np.concatenate([np.arange(a, b + 1) for a, b in zip(first, last)]).tolist())


class _Rows:
    """Operand rows read from a backend: name -> (sorted rows, values); a BoundSim reader with bound 0."""

    def __init__(self):
        self.d = {}

    def __call__(self, name, rows):
        have, vals = self.d[name]
        pos = np.searchsorted(have, rows)
        assert np.array_equal(have[np.minimum(pos, len(have) - 1)], rows), f'operand {name}: rows not read'
        v = vals[pos].astype(np.float64)
        return v, np.zeros_like(v)


class Failure(AssertionError):
    pass


class _done:
    """A finished result with the Future interface."""

    def __init__(self, value):
        self.value = value

    def result(self):
        return self.value


class Sweep:
    """One program, op by op.  ``pb``: the lowered plan; ``blob``: its weight arena; ``engines``: the engine each op
    resolves to; ``backend``: see the module docstring.  ``interior``: seeded interior rows per sampled M tile."""

    def __init__(self, name, pb, blob, engines, backend, seed=0, interior=1, ops=None):
        self.name, self.pb, self.backend = name, pb.finalize(), backend
        self.engines = list(engines)
        self.sim = eb.BoundSim.for_ops(self.pb, blob, self.engines)
        rng = np.random.default_rng(seed)
        self.kernels = [oc.kernel_of(o, e) for o, e in zip(self.pb.ops, self.engines)]
        self.rows = [sample_rows(o, e, k, rng, interior) for o, e, k in zip(self.pb.ops, self.engines, self.kernels)]
        self.ops = range(len(self.pb.ops)) if ops is None else ops
        self.slot_max = {}
        self.stats = {}                       # kernel -> [worst ratio, checked elements]
        self._lock = threading.Lock()

    def _read_operands(self, i):
        o = self.pb.ops[i]
        v = eb.views(o)
        got = _Rows()
        for name, rows in eb.operand_rows(o, self.rows[i]).items():
            got.d[name] = (rows, self.backend.rows(v[name], rows))
        return got

    def run(self, workers=1, log=None):
        """Every op's check; raises Failure for the first op (in program order) above its bound.  With ``workers`` > 1
        the references run on a thread pool while the backend runs the next prefixes."""
        operands = self._read_operands(0)
        last = max(self.ops)
        pending = []
        with ThreadPoolExecutor(max(1, workers)) as pool:
            try:
                for i in range(last + 1):
                    o = self.pb.ops[i]
                    if log is not None:
                        log(i)
                    self.backend.run(prefix(self.pb, i))
                    v = eb.views(o)
                    if o.amax_out > 0:
                        self.slot_max[o.amax_out] = max(self.slot_max.get(o.amax_out, 0.0),
                                                        self.backend.amax(v['dst']))
                    outs = {name: self.backend.rows(v[name], self.rows[i]) for name in ('dst', 'sum') if name in v}
                    nxt = self._read_operands(i + 1) if i < last else None
                    if i in self.ops:
                        s = self.scale_exp(i)
                        pending.append(pool.submit(self.check, i, operands, outs, s) if workers > 1
                                       else _done(self.check(i, operands, outs, s)))
                    operands = nxt
            finally:
                self.backend.close()
            for j, f in zip(self.ops, pending):
                f.result()
                if log is not None:
                    log(j)
        return self.stats

    def scale_exp(self, i):
        o = self.pb.ops[i]
        if self.engines[i] != L.ENGINE_TC16:
            return 0
        return eb.design_scale_exp(self.slot_max.get(o.amax_in, 0.0))

    def reference(self, i, operands, s=None):
        sim = copy.copy(self.sim)                             # one per call: ``i`` selects the engine
        sim.i = i
        return sim.op(self.pb.ops[i], self.rows[i], operands, self.scale_exp(i) if s is None else s)

    def check(self, i, operands, outs, s=None):
        o, k = self.pb.ops[i], self.kernels[i]
        ref = self.reference(i, operands, s)
        for name, got in outs.items():
            want, beta = ref[name]
            got = got.astype(np.float64)
            d = np.abs(got - want)
            with np.errstate(invalid='ignore', divide='ignore'):
                r = np.where(beta > 0, d / np.where(beta > 0, beta, 1.0), np.where(d > 0, np.inf, 0.0))
            r = np.where(np.isfinite(want) & ~np.isfinite(got), np.inf, r)
            r = np.where(np.isnan(r), np.inf, r)
            worst = float(r.max()) if r.size else 0.0
            with self._lock:
                s = self.stats.setdefault(k, [0.0, 0])
                s[0], s[1] = max(s[0], worst), s[1] + r.size
            if not worst <= 1.0:
                j, n = np.unravel_index(int(np.argmax(r)), r.shape)
                m = int(self.rows[i][j])
                where = locate(o, self.engines[i], k, m, int(n))
                raise Failure(f'{self.name} op {i} ({k}) {name}: err/beta {worst:.3g} at row {m}, column {int(n)}'
                              + ''.join(f', {a} {b}' for a, b in where.items())
                              + f': got {got[j, n]!r}, fp64 {want[j, n]!r}, bound {beta[j, n]:.3g}')


# ---------------------------------------------------------------------------------------------------------------
# backends
# ---------------------------------------------------------------------------------------------------------------
class GpuBackend:
    """The library on the GPU: each prefix is a Program run once, eagerly (vp_embed), on the same input; views are
    read with vp_program_peek into device memory, and only the sampled rows go to the host."""

    def __init__(self, blob, feats):
        import torch
        from mvector.engine import Engine
        self.torch = torch
        self.eng = Engine()
        self.eng.load_weights(blob)
        self.feats = feats.contiguous().view(-1)
        self.prog = None
        self.emb = None
        self.cache = {}

    def run(self, pb):
        from mvector.engine import Program
        if self.prog is not None:
            self.prog.close()
        self.cache = {}
        if self.emb is None:
            self.emb = self.torch.full((pb.out_floats,), float('nan'), device='cuda')
        self.prog = Program(self.eng, pb)
        self.prog.run(self.feats, self.emb)
        self.torch.cuda.synchronize()

    def _view(self, view):
        import ctypes as C
        torch = self.torch
        off, ld, coff, Cn, rows = view
        key = (off, ld, coff, Cn, rows)
        if key not in self.cache:
            if off == L.BUF_INPUT:
                flat = self.feats
            elif off == L.BUF_OUTPUT:
                flat = self.emb
            else:
                n = (rows - 1) * ld + coff + Cn
                flat = torch.empty(rows * ld, dtype=torch.float32, device='cuda')
                rc = L.lib().vp_program_peek(self.prog._p, off, n * 4, C.c_void_p(flat.data_ptr()),
                                             self.eng.stream_ptr())
                assert rc == 0, rc
                torch.cuda.synchronize()
            self.cache = {key: flat.view(rows, ld)[:, coff:coff + Cn]}     # the last view read: keep one at a time
        return self.cache[key]

    def rows(self, view, rows):
        t = self._view(view)
        return t[self.torch.from_numpy(np.asarray(rows, dtype=np.int64)).cuda()].cpu().numpy()

    def amax(self, view):
        return float(self._view(view).abs().max())

    def close(self):
        if self.prog is not None:
            self.prog.close()
            self.prog = None
        self.eng.close()


class SimBackend:
    """The fp64 interpreter (plan_sim.Sim, fp32 storage) standing in for the GPU: each prefix extends the one before it
    by its new ops.  ``mutate(self, i, o)`` runs op i in place of Sim (see tests/test_bench_programs_cpu.py)."""

    def __init__(self, pb, blob, feats, mutate=None):
        from plan_sim import Sim
        self.sim = Sim(pb, blob, feats)
        self.done = []
        self.mutate = mutate

    def run(self, pb):
        assert [id(o) for o in pb.ops[:len(self.done)]] == [id(o) for o in self.done], 'not a prefix of the last run'
        s = self.sim
        for o in pb.ops[len(self.done):]:
            i = len(self.done)
            if self.mutate is None or not self.mutate(self, i, o):
                {L.OP_CONV: s.conv, L.OP_CONV_C1: s.conv, L.OP_COLSTATS: s.colstats, L.OP_ASP_POOL: s.asp,
                 L.OP_EW: s.ew, L.OP_POOL2D: s.pool2d}[o.kind](o)
            self.done.append(o)

    def _idx(self, view, rows):
        off, ld, coff, Cn, _ = view
        mem, base = self.sim._mem(off)
        return mem, base + np.asarray(rows)[:, None] * ld + coff + np.arange(Cn)[None, :]

    def rows(self, view, rows):
        mem, idx = self._idx(view, rows)
        return mem[idx].copy()

    def amax(self, view):
        mem, idx = self._idx(view, np.arange(view[4]))
        return float(np.abs(mem[idx]).max())

    def close(self):
        pass
