"""Ragged case table for the op-level tests of vp_features_each (tests/test_gpu_frontend_each_edges.py on the GPU,
tests/test_frontend_each_cases_cpu.py on the CPU): one ragged batch per case of tests/frontend_cases.py.

The longest row keeps the case's T, so the call runs the plan the case names (its ``intent``).  The other rows sit on
the ragged edges of that plan: the shortest row a one-row call accepts, T_b = 15 / 0 / 1 mod 16, T_b = 16 tpc -+ 1 (a
row's last live tile sharing its CTA with dead tiles), T_b = T - 1 and lengths off the hop grid; the longest row is
neither first nor last.  The stride is ld = Lmax + d with d odd and Lmax even, so the rows start at every 16-byte
residue and every row has a tail; in the WIDE cases ld is far past Lmax and the call's T = num_frames(ld) exceeds every
row's T_b.  MFCC rows differ in gain (a quiet row, and a loud row whose bursts sit > 80 dB above its pauses), so every
row's top_db clamp differs from the whole call's.

``length_ok`` restates csrc/api.cu's one-row length check (frontend_length_error + at least one frame).
Never imported by the product."""
import numpy as np

import frontend_cases as fc
from mvector import _lib as L

# case -> frames the stride reaches past the longest row (T = num_frames(ld) = the case's T + this); the plan of those
# cases is kept at its intent because their tpc is already 4, or held at 1 by shared memory
WIDE = {'fbank80_512_tpc1_residues': 40, 'mel40_256_tpc4_constant': 37, 'mel40_200_tpc4_nocenter_pad': 41,
        'mfcc_256_tpc4': 35}
POISONS = (float('nan'), float('inf'), float('-inf'), 3e38)   # the tail value wave[b, lens[b]:ld] of case i: POISONS[i % 4]
QUIET, LOUD, PAUSE = 1e-3, 30.0, 3e-4                          # MFCC row gains: LOUD / PAUSE = 100 dB


def length_ok(fz, n):
    """Whether a one-row call takes n samples: api.cu frontend_length_error(n) == "" and vp_num_frames(n) >= 1."""
    f = fz.feat_fun
    o, half = f.opts, f.n_fft // 2
    Lp = n + 2 * o.pad
    if f.desc.kind == 0:
        ok = 2 <= f.win_length <= n
    elif o.frame_mode == L.FRAME_DEFAULT:
        ok = half < Lp
    elif o.frame_mode == L.FRAME_STFT_CIRCULAR:
        ok = half <= Lp
    elif o.frame_mode == L.FRAME_STFT_NOCENTER:
        ok = f.n_fft <= Lp
    else:
        ok = n >= 1
    return ok and fz.num_frames(n) >= 1


def shortest_row(fz):
    """The fewest samples a one-row call accepts (every length rule holds from some minimum up)."""
    n = 0
    while not length_ok(fz, n):
        n += 1
    return n


def _row_frames(T, tpc, Tmin):
    """The T_b < T of the ragged edges, each kept only where T allows it."""
    want = {Tmin, T - 1, 16 * tpc - 1, 16 * tpc + 1}
    for r in (15, 0, 1):                                   # the largest T_b below T at each tile residue
        t = (T - 1) - ((T - 1 - r) % 16)
        want.add(t)
    return sorted(t for t in want if max(Tmin, 1) <= t < T)


def build(name):
    """-> dict(method, args, intent, wave [B, ld] float32 (tails poisoned), lens [B], ld, T (the call's frames),
    n (the length whose frames are T: the plan's), Tb [B], Lmax, longest (row index), poison, wide)."""
    c = fc.CASES[name]
    method, args, T0 = c['method'], c['args'], c['T']
    fz = fc.featurizer(method, args)
    f = fz.feat_fun
    hop = f.hop
    rng = np.random.default_rng(sum(map(ord, name)) + 1)
    tpc = fc.plan_of(name)['tpc']
    n_min = shortest_row(fz)
    Tmin = fz.num_frames(n_min)

    # the longest row: T0 frames, an even length, room for an odd d before the stride leaves T0's frames
    e = min(c.get('extra', 0), hop - 2)
    if fc.lpad_for(method, args, T0, e) % 2:
        e = e + 1 if e + 1 <= hop - 2 else e - 1
    Lmax = fc.lpad_for(method, args, T0, e)
    d = 1 + 2 * int(rng.integers(0, (hop - 1 - e + 1) // 2))      # odd, 1 <= d <= hop - 1 - e
    ld = Lmax + d
    assert fz.num_frames(ld) == T0 and d % 2 == 1 and ld % 2 == 1
    wide = name in WIDE
    if wide:
        ld = fc.lpad_for(method, args, T0 + WIDE[name])
        ld += (ld - Lmax + 1) % 2                                  # ld - Lmax odd
    T = fz.num_frames(ld)

    lens = [n_min]
    for tb in _row_frames(T0, tpc, Tmin):
        if tb == Tmin:
            continue
        for ex in (int(rng.integers(1, hop)), 0):                  # off the hop grid where T_b allows it
            n = max(fc.lpad_for(method, args, tb, ex), n_min)
            if fz.num_frames(n) == tb and length_ok(fz, n):
                lens.append(n)
                break
    if len(lens) < 2:                                              # T0 = 1: a second row of T0 frames
        lens.append((n_min + Lmax) // 2)
    order = rng.permutation(len(lens) - 1) + 1                     # the shortest row first, the rest shuffled
    lens = [lens[0]] + [lens[i] for i in order]
    longest = (len(lens) + 1) // 2                                 # neither first nor last
    lens.insert(longest, Lmax)
    B = len(lens)

    # rows: 0.1 N(0, 1) times a per-row gain; MFCC: the shortest row quiet, the longest loud in bursts over pauses
    x = np.zeros((B, ld), np.float32)
    poison = POISONS[list(fc.CASES).index(name) % len(POISONS)]
    for b, n in enumerate(lens):
        if f.desc.post == 1:
            if b == longest:
                g = np.resize(np.repeat([LOUD, PAUSE], 8 * hop), n)
            else:
                g = QUIET if b == 0 else 1.0
        else:
            g = float(np.exp(rng.uniform(np.log(0.05), np.log(2.0))))
        x[b, :n] = g * 0.1 * rng.standard_normal(n)
        x[b, n:] = poison
    return dict(method=method, args=args, intent=c['intent'], wave=x, lens=lens, ld=ld, T=T, n=ld if wide else Lmax,
                Tb=[fz.num_frames(n) for n in lens], Lmax=Lmax, longest=longest, poison=poison, wide=wide, tpc=tpc,
                n_min=n_min)


def plan_of(case):
    """The host-plan mirror of the ragged call: the plan of T = num_frames(n) frames."""
    return fc.frontend_plan(fc.geometry(case['method'], case['args']), -(-case['T'] // fc.FPB))


CASES = list(fc.CASES)
