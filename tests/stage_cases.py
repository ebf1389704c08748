"""Case tables and launch-plan mirrors for the op-level tests of the input conditioning (csrc/condition.cu) and the
diarization spectral stage (csrc/spectral.cu): tests/test_gpu_stage_edges.py on the GPU, tests/test_stage_cases_cpu.py
on the CPU.

Each case records the launch path it is meant to reach (``intent``).  The mirrors below restate the kernels' host-side
and per-CTA decisions, so the CPU suite can check that every case really lands where it claims:
  - ``resample_ctas``: which CTAs of a resample row stage their input window in shared memory and which read global
    memory (resample_kernel's ``staged`` predicate, condition.cu:72-75);
  - ``pass_grid`` / ``spectral_plan``: the row tiling of tridiag_pass_kernel, how many ``rb`` chunks a CTA stages, the
    prune kernel's dynamic shared memory and the apply_q size limit (spectral.cu:321-329, 409-414, 443-445, api.cu:881).
Never imported by the product."""
import numpy as np

from mvector.audio import resample_ratio, resampled_length

# ---------------------------------------------------------------------------------------------------------------
# resampler (csrc/condition.cu)
# ---------------------------------------------------------------------------------------------------------------
RS_THREADS = 256                                  # output samples per CTA
RS_WINDOW = 4096                                  # staged input samples per CTA
GN_TILE = 256 * 16                                # samples per energy partial of the gain


def rs_filter(up, down):
    """condition.cu rs_filter -> (Lh, nt, n_pre_remove)."""
    max_rate = max(up, down)
    half_len = 10 * max_rate
    n_pre_pad = down - half_len % down
    Lh = n_pre_pad + 2 * half_len + 1
    return Lh, -(-Lh // up), (half_len + n_pre_pad) // down


def rs_kmin(t0, Lh, up):
    """condition.cu rs_kmin: the first input sample under output t0's filter."""
    num = t0 - (Lh - 1)
    return 0 if num <= 0 else -(-num // up)


def resample_ctas(n_in, rate, target):
    """CTAs of one row that hold outputs -> (staged, global_read); (0, 0) for a copy row (rate == target).  CTAs past
    n_out only write padding and are not counted."""
    up, down = resample_ratio(rate, target)
    if up == down:
        return 0, 0
    n_out = int(resampled_length(n_in, up, down))
    Lh, _, npr = rs_filter(up, down)
    staged = glob = 0
    for j0 in range(0, n_out, RS_THREADS):
        j_last = min(j0 + RS_THREADS, n_out) - 1
        w_lo = rs_kmin((j0 + npr) * down, Lh, up)
        w_hi = min(n_in - 1, (j_last + npr) * down // up)
        if w_hi - w_lo + 1 <= RS_WINDOW:
            staged += 1
        else:
            glob += 1
    return staged, glob


def intent_class(counts):
    staged, glob = counts
    if staged == glob == 0:
        return 'copy'
    return 'staged' if glob == 0 else ('global' if staged <= 1 else 'mixed')


def n_in_for(rate, target, n_out):
    """The smallest input length whose resampled length is n_out."""
    up, down = resample_ratio(rate, target)
    n = max(1, (n_out - 1) * down // up)
    while int(resampled_length(n, up, down)) < n_out:
        n += 1
    assert int(resampled_length(n, up, down)) == n_out
    return n


def _rs(rate, n_in, staged, glob, target=16000, name=None):
    return dict(name=name or f'{rate}->{target}_n{n_in}', rate=rate, target=target, n_in=n_in, intent=(staged, glob))


# intent = (staged CTAs, global-read CTAs).  The input window of one CTA is about 275 down / up samples, so down <= 14
# stages every CTA and down >= 15 reads global memory in all but the edge CTAs, whose window is clipped at 0 or n_in.
RESAMPLE_CASES = [
    _rs(16000, 48007, 0, 0, name='copy_16k'),
    _rs(44100, 3 * 44100 + 7, 188, 0, name='staged_44k1_3s'),
    _rs(224000, 3 * 224000, 188, 0, name='staged_224k_3s'),                  # down = 14: the last fully staged ratio
    _rs(240000, 3 * 240000, 2, 186, name='mixed_240k_3s'),                   # down = 15: both edge CTAs staged
    _rs(256000, 3 * 256000, 1, 187, name='global_256k_3s'),
    _rs(384000, 3 * 384000, 1, 187, name='global_384k_3s'),
    _rs(352800, 3 * 352800, 1, 187, name='global_352k8_3s'),                 # 20 / 441
    _rs(7350, 3 * 7350, 188, 0, name='upsample_7350_3s'),                    # 320 phases
    # n_out = 256 j - 1, 256 j, 256 j + 1: the last CTA holds 255, 256 or 1 outputs
    _rs(240000, n_in_for(240000, 16000, 8 * 256 - 1), 2, 6, name='mixed_240k_nout2047'),
    _rs(240000, n_in_for(240000, 16000, 8 * 256), 2, 6, name='mixed_240k_nout2048'),
    _rs(240000, n_in_for(240000, 16000, 8 * 256 + 1), 3, 6, name='mixed_240k_nout2049'),
    _rs(384000, n_in_for(384000, 16000, 20 * 256 - 1), 0, 20, name='global_384k_nout5119'),
    _rs(384000, n_in_for(384000, 16000, 20 * 256), 0, 20, name='global_384k_nout5120'),
    _rs(384000, n_in_for(384000, 16000, 20 * 256 + 1), 1, 20, name='global_384k_nout5121'),
    _rs(44100, n_in_for(44100, 16000, 12 * 256 - 1), 12, 0, name='staged_44k1_nout3071'),
    _rs(44100, n_in_for(44100, 16000, 12 * 256), 12, 0, name='staged_44k1_nout3072'),
    _rs(44100, n_in_for(44100, 16000, 12 * 256 + 1), 13, 0, name='staged_44k1_nout3073'),
    # rows shorter than the filter half-length (10 down = 240 input samples at 384 kHz): every output's window is clipped
    _rs(384000, 1, 1, 0, name='short_384k_n1'),
    _rs(384000, 5, 1, 0, name='short_384k_n5'),
    _rs(384000, 64, 1, 0, name='short_384k_n64'),
    _rs(240000, 239, 1, 0, name='short_240k_n239'),
    # other targets, one call each
    _rs(48000, 3 * 48000 + 5, 94, 0, target=8000, name='48k->8k'),
    _rs(384000, 3 * 384000, 0, 94, target=8000, name='384k->8k'),
    _rs(44100, 2 * 44100 + 3, 63, 0, target=8000, name='44k1->8k'),
    _rs(8000, 2 * 8000 + 1, 376, 0, target=48000, name='8k->48k'),
    _rs(44100, 2 * 44100 + 1, 376, 0, target=48000, name='44k1->48k'),
    _rs(16000, 16001, 188, 0, target=48000, name='16k->48k'),
]
RESAMPLE_TARGETS = sorted({c['target'] for c in RESAMPLE_CASES})


# ---------------------------------------------------------------------------------------------------------------
# gain (csrc/condition.cu)
# ---------------------------------------------------------------------------------------------------------------
def _gn(name, n, amp, max_gain_db=300.0, flagged=False, inf_at=None):
    return dict(name=name, n=n, amp=amp, max_gain_db=max_gain_db, flagged=flagged, inf_at=inf_at)


# Rows of one max_gain_db run in one call, at 16 kHz (no resampling): the gain works in place on rows of a leading
# dimension ld >= 3 GN_TILE beyond the longest row.  ``flagged``: AudioSegment.normalize raises and the row stays as it
# was.  1e-20 full scale is -400 dB: a gain of 380 dB.  One inf sample makes the mean inf, the gain -inf and the factor
# 0: the row becomes signed zeros with a NaN at the inf.
GAIN_CASES = [
    _gn('n1', 1, 0.3),
    _gn('n4095', GN_TILE - 1, 0.2),
    _gn('n4096', GN_TILE, 0.05),
    _gn('n4097', GN_TILE + 1, 0.4),
    _gn('n8192', 2 * GN_TILE, 0.1),
    _gn('n12289', 3 * GN_TILE + 1, 0.02),
    _gn('quiet_1e-20', 3 * GN_TILE + 1, 1e-20, flagged=True),
    _gn('inf_sample', 2 * GN_TILE + 17, 0.1, inf_at=GN_TILE + 5),
    _gn('max10_loud_n4097', GN_TILE + 1, 0.5, max_gain_db=10.0),
    _gn('max10_quiet_n4097', GN_TILE + 1, 0.01, max_gain_db=10.0, flagged=True),
    _gn('max10_quiet_n1', 1, 0.01, max_gain_db=10.0, flagged=True),
    _gn('max10_loud_n8192', 2 * GN_TILE, 0.3, max_gain_db=10.0),
    _gn('max10_quiet_n12289', 3 * GN_TILE + 1, 0.003, max_gain_db=10.0, flagged=True),
]
GAIN_PAD_TILES = 3


def gain_rows(cases, seed):
    """Deterministic float32 rows for gain cases: amplitude ``amp`` times a standard normal, a -0 and a +0 planted in
    rows of 8 samples or more (their signs must survive the scaling), and the inf."""
    rng = np.random.default_rng(seed)
    rows = []
    for c in cases:
        x = (rng.standard_normal(c['n']) * c['amp']).astype(np.float32)
        if c['n'] >= 8:
            x[3], x[c['n'] - 2] = -0.0, 0.0
        if c['inf_at'] is not None:
            x[c['inf_at']] = np.inf
        rows.append(x)
    return rows


def host_normalize(x, target_db, max_gain_db):
    """AudioSegment.normalize -> (row, flagged): a row it refuses is flagged and kept as it was."""
    from mvector.audio import AudioSegment
    seg = AudioSegment(x.copy(), 16000)
    try:
        with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
            seg.normalize(target_db=target_db, max_gain_db=max_gain_db)
    except ValueError:
        return x, True
    return seg.samples, False


# ---------------------------------------------------------------------------------------------------------------
# spectral stage (csrc/spectral.cu)
# ---------------------------------------------------------------------------------------------------------------
PASS_THREADS = 256
PASS_GY_MAX = 32
SMS = 132
APPLYQ_CTAS = 8
STATIC_SMEM = 48 * 1024                           # above this a kernel needs the dynamic shared memory opt-in
OPTIN_SMEM = 227 * 1024


def pass_grid(m):
    """spectral.cu pass_grid over an m x m trailing block -> (gx, gy, rows_per)."""
    gx = -(-m // PASS_THREADS)
    g = min(-(-(8 * SMS) // gx), PASS_GY_MAX, m)
    g = max(g, 1)
    rows_per = -(-m // g)
    return gx, -(-m // rows_per), rows_per


def apply_q_max_rows(kz):
    """spectral.cu apply_q_max_rows: rows of Z per CTA that fit in the opt-in shared memory."""
    return (OPTIN_SMEM // 8 - 32) // (kz + 1)


def apply_q_max_n(kz):
    """The largest n vp_sym_tridiag_apply_q accepts at kz columns (api.cu:881)."""
    return APPLYQ_CTAS * apply_q_max_rows(kz)


def apply_q_smem(n, kz):
    R = -(-n // APPLYQ_CTAS)
    return (32 + R * (kz + 1)) * 8


def spectral_plan(n, kz=16):
    """Launch decisions at size n: the first pass (k = 0, trailing block n - 1), its ``rb`` chunks per CTA, the prune
    kernel's dynamic shared memory and whether apply_q accepts [n, kz]."""
    gx, gy, rows_per = pass_grid(n - 1)
    return dict(gy=gy, rows_per=rows_per, chunks=-(-rows_per // PASS_THREADS),
                prune_optin=n * 4 > STATIC_SMEM, apply_q_ok=-(-n // APPLYQ_CTAS) <= apply_q_max_rows(kz))


def _sp(n, gy, rows_per, chunks, prune_optin, apply_q_ok=True, kz=16):
    return dict(name=f'n{n}', n=n, kz=kz, intent=dict(gy=gy, rows_per=rows_per, chunks=chunks, prune_optin=prune_optin,
                                                      apply_q_ok=apply_q_ok))


SPECTRAL_CASES = [
    _sp(8450, 32, 265, 2, False),                 # every CTA stages two rb chunks, all 32 row tiles
    _sp(12288, 22, 559, 3, False),                # the prune row is exactly 48 KB: no opt-in
    _sp(12289, 22, 559, 3, True),                 # the first size with the prune opt-in
    _sp(13656, 20, 683, 3, True),                 # apply_q's limit at k = 16: 232 408 B of shared memory
]
APPLY_Q_REFUSED = dict(n=13657, kz=16, accepted_kz=2)


# Components of the permuted block-diagonal Laplacians of the tridiagonal-stage tests: three unequal blocks per size,
# drawn from one pool so the reference spectra (per-block eigvalsh) are computed once per block.
BLOCK_POOL = (4763, 4552, 4341, 3396, 502)
TRIDIAG_BLOCKS = {8450: (4552, 3396, 502), 12289: (4552, 4341, 3396), 13656: (4763, 4552, 4341)}
