"""Op-level tests of the input conditioning (csrc/condition.cu) and the diarization spectral stage (csrc/spectral.cu)
at the launch-path switches the comfortable sizes never cross (tests/stage_cases.py names each case's path):
  - the resampler's global-read loop, and rows of one launch whose CTAs take different loops, bit-identical to
    AudioSegment.resample; targets other than 16 kHz;
  - the gain at GN_TILE boundaries, with ld tiles beyond the row, a custom max_gain_db, a 380 dB row and an inf sample,
    bit-identical to AudioSegment.normalize;
  - the Laplacian where the prune row needs the dynamic shared memory opt-in;
  - the Householder reduction where a pass CTA stages several row chunks and the row tiles drop below 32, up to
    apply_q's size limit, against per-block eigenvalues of a permuted block-diagonal Laplacian and the trace /
    Frobenius invariants of the whole spectrum;
  - apply_q's refusal one past that limit."""
import numpy as np
import pytest
import scipy.linalg
import torch

import stage_cases as sc
from oracle import spectral as osp
from test_gpu_spectral import _check_laplacian, _clustered, _device_eig

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from mvector.engine import Engine
    e = Engine()
    yield e
    e.close()


# ------------------------------------------------------------------------------------------------ resampler
def _host_resample(x, rate, target):
    from mvector.audio import AudioSegment
    seg = AudioSegment(x.copy(), rate)
    seg.resample(target)
    return seg.samples


def _resample_launch(eng, cases, target, seed):
    """One vp_resample launch over ``cases``: input rows NaN past n_in (a read beyond the row poisons its outputs),
    output NaN-poisoned with out_ld past every n_out.  -> (native rows, n_out, y numpy)."""
    rng = np.random.default_rng(seed)
    waves = [(rng.standard_normal(c['n_in']) * rng.uniform(0.05, 0.5)).astype(np.float32) for c in cases]
    n_in = [c['n_in'] for c in cases]
    in_ld = max(n_in) + 37
    x = np.full((len(cases), in_ld), np.nan, dtype=np.float32)
    for i, w in enumerate(waves):
        x[i, :w.size] = w
    plan = eng.condition_plan(n_in, [c['rate'] for c in cases], target)
    assert plan.resample and not plan.gain
    out_ld = int(plan.n_out.max()) + 2 * sc.RS_THREADS + 3
    xd = torch.from_numpy(x).cuda()

    def run():
        y = torch.full((len(cases), out_ld), float('nan'), dtype=torch.float32, device='cuda')
        plan.run(xd, in_ld, y, out_ld, 0, len(cases), None, None)
        return y.cpu().numpy()

    y = run()
    assert np.array_equal(run().view(np.uint32), y.view(np.uint32))          # two calls bit-identical
    return waves, plan.n_out, y


def _check_resampled(cases, waves, n_out, y, target):
    for i, (c, w) in enumerate(zip(cases, waves)):
        ref = _host_resample(w, c['rate'], target)
        assert n_out[i] == ref.size, c['name']
        assert np.array_equal(y[i, :ref.size], ref), (c['name'], int(np.sum(y[i, :ref.size] != ref)))
        assert not y[i, ref.size:].view(np.uint32).any(), c['name']            # padding exactly +0


def test_resample_every_path_in_one_launch(eng):
    """Copy, staged, mixed and global-read rows together: CTAs of one launch, and of one row, take different loops."""
    cases = [c for c in sc.RESAMPLE_CASES if c['target'] == 16000]
    assert {sc.intent_class(c['intent']) for c in cases} == {'copy', 'staged', 'mixed', 'global'}
    waves, n_out, y = _resample_launch(eng, cases, 16000, seed=1)
    _check_resampled(cases, waves, n_out, y, 16000)


@pytest.mark.parametrize('target', [t for t in sc.RESAMPLE_TARGETS if t != 16000])
def test_resample_other_targets(eng, target):
    cases = [c for c in sc.RESAMPLE_CASES if c['target'] == target]
    waves, n_out, y = _resample_launch(eng, cases, target, seed=target)
    _check_resampled(cases, waves, n_out, y, target)


# ------------------------------------------------------------------------------------------------ gain
def _same_bits_nan_aware(got, ref):
    """NaN at the same positions, every other sample bit for bit (the sign of zero included)."""
    nan = np.isnan(ref)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32))


@pytest.mark.parametrize('max_gain_db', sorted({c['max_gain_db'] for c in sc.GAIN_CASES}))
def test_gain_edges_bit_identical_to_normalize(eng, max_gain_db):
    cases = [c for c in sc.GAIN_CASES if c['max_gain_db'] == max_gain_db]
    rows = sc.gain_rows(cases, seed=int(max_gain_db))
    lens = [c['n'] for c in cases]
    ld = max(lens) + sc.GAIN_PAD_TILES * sc.GN_TILE + 5
    x = np.full((len(cases), ld), 7.0, dtype=np.float32)                     # past n: neither summed nor scaled
    for i, w in enumerate(rows):
        x[i, :w.size] = w
    xd = torch.from_numpy(x).cuda()
    y, n_out, flags = eng.condition(xd, lens, 16000, 16000, target_db=-20, max_gain_db=max_gain_db)
    y, fl = y.cpu().numpy(), flags.cpu().numpy()
    for i, (c, w) in enumerate(zip(cases, rows)):
        ref, flag = sc.host_normalize(w, -20, max_gain_db)
        assert fl[i] == int(flag) and flag == c['flagged'], c['name']
        assert _same_bits_nan_aware(y[i, :c['n']], ref), (c['name'], int(np.sum(y[i, :c['n']] != ref)))
        assert (y[i, c['n']:] == 7.0).all(), c['name']
    y2, _, fl2 = eng.condition(xd, lens, 16000, 16000, target_db=-20, max_gain_db=max_gain_db)
    assert np.array_equal(y2.cpu().numpy().view(np.uint32), y.view(np.uint32))
    assert np.array_equal(fl2.cpu().numpy(), fl)


# ------------------------------------------------------------------------------------------------ Laplacian
@pytest.mark.parametrize('n', [c['n'] for c in sc.SPECTRAL_CASES if c['intent']['prune_optin']])
def test_laplacian_with_prune_smem_opt_in(eng, n):
    _check_laplacian(eng, _clustered(n, seed=n))


# ------------------------------------------------------------------------------------------------ eigen stage
@pytest.fixture(scope='module')
def blocks():
    """Block Laplacian and its 16 smallest eigenvalues for every size of sc.BLOCK_POOL, computed once."""
    out = {}
    for m in sc.BLOCK_POOL:
        Lb = osp.laplacian(osp.prune(osp.cosine(_clustered(m, seed=m)), osp.n_drop(m)))
        out[m] = (Lb, scipy.linalg.eigh(Lb, eigvals_only=True, subset_by_index=[0, 15]))
    return out


@pytest.mark.parametrize('n', sorted(sc.TRIDIAG_BLOCKS))
def test_tridiag_past_one_row_chunk(eng, blocks, n):
    """Three disconnected components, interleaved by a permutation: the 16 smallest eigenvalues are those of the
    union of the blocks' spectra (0 three times), the invariants sum(d) = trace(L) and sum(d^2) + 2 sum(e^2) =
    ||L||_F^2 see every reflector of the reduction."""
    parts = sc.TRIDIAG_BLOCKS[n]
    Lh = scipy.linalg.block_diag(*[blocks[m][0] for m in parts])
    perm = np.random.RandomState(n).permutation(n)
    Lh = np.ascontiguousarray(Lh[perm][:, perm])
    lam_ref = np.sort(np.concatenate([blocks[m][1] for m in parts]))[:16]
    Ld = torch.from_numpy(Lh).cuda()
    d1, e1, lam, Z1 = _device_eig(eng, Ld, 16)
    norm1 = np.abs(Lh).sum(axis=0).max()
    tr, fro2 = np.trace(Lh), np.sum(Lh * Lh)
    err = dict(lam=np.abs(lam[:16] - lam_ref).max() / norm1, res=np.abs(Lh @ Z1 - Z1 * lam[:16]).max() / norm1,
               orth=np.abs(Z1.T @ Z1 - np.eye(16)).max(), trace=abs(d1.sum() - tr) / abs(tr),
               fro=abs(np.sum(d1 * d1) + 2.0 * np.sum(e1 * e1) - fro2) / fro2)
    print(f'n = {n}: ' + ', '.join(f'{k} {v:.1e}' for k, v in err.items()))
    assert np.abs(lam[:3]).max() <= 1e-10 * norm1
    assert err['lam'] <= 1e-10 and err['res'] <= 1e-9 and err['orth'] <= 1e-10, err
    assert err['trace'] <= 1e-12 and err['fro'] <= 1e-12, err
    d2, e2, _, Z2 = _device_eig(eng, Ld, 16)                        # bit-reproducible
    assert np.array_equal(d1, d2) and np.array_equal(e1, e2) and np.array_equal(Z1, Z2)


def test_apply_q_refused_past_its_limit(eng):
    """n = 8 apply_q_max_rows(16) + 1 at k = 16 does not fit the cluster's shared memory: VP_ERR_UNSUPPORTED before
    anything is launched.  At k = 2 the same n runs; with every tau 0, Q = I and Z comes back bit for bit."""
    from mvector import _lib as L
    r = sc.APPLY_Q_REFUSED
    n = r['n']
    A = torch.zeros(n, n, dtype=torch.float64, device='cuda')
    tau = torch.zeros(n - 1, dtype=torch.float64, device='cuda')
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        with pytest.raises(L.VpError) as ei:
            eng.sym_tridiag_apply_q(A, tau, np.zeros((n, r['kz'])))
        torch.cuda.synchronize()
    assert ei.value.code == L.VP_ERR_UNSUPPORTED
    assert not [ev.name for ev in prof.events() if 'apply_q' in ev.name]
    Z = np.random.default_rng(0).standard_normal((n, r['accepted_kz']))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        got = eng.sym_tridiag_apply_q(A, tau, Z).cpu().numpy()
    assert [ev.name for ev in prof.events() if 'apply_q' in ev.name]        # the trace does see the kernel
    assert np.array_equal(got, Z)
