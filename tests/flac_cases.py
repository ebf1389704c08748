"""FLAC streams shared by the CPU and GPU tests: a seeded matrix over the frame and subframe features of RFC 9639, each
stream with the integer PCM it encodes."""
import numpy as np

import flac_writer as fw


def _kinds(kind_cycle, order_cycle, prec=12, shift=None, part_order=0, method_cycle=(0,), esc_cycle=((),), wasted=0):
    def sub(fi, c, x):
        k = kind_cycle[(fi + c) % len(kind_cycle)]
        kw = dict(kind=k, method=method_cycle[(fi + c) % len(method_cycle)], wasted=wasted)
        if k in ('fixed', 'lpc'):
            order = min(order_cycle[(fi + c) % len(order_cycle)], len(x), 4 if k == 'fixed' else 32)
            order = max(order, 1 if k == 'lpc' else 0)
            po = part_order
            while po and ((len(x) >> po) << po != len(x) or (len(x) >> po) < order):
                po -= 1
            esc = tuple(p for p in esc_cycle[(fi + c) % len(esc_cycle)] if p < (1 << po))
            kw.update(order=order, prec=prec, part_order=po, escape_parts=esc)
            if shift is not None:
                kw['shift'] = shift
        if k == 'constant' and len(set(int(v) for v in x)) != 1:
            kw['kind'] = 'verbatim'
        return kw
    return sub


def matrix(seed=0):
    """[(name, flac bytes, pcm int64 [n, ch], bps)]"""
    rng = np.random.default_rng(seed)
    out = []

    def add(name, pcm, bps, **kw):
        out.append((name, fw.encode(pcm, kw.pop('rate', 16000), bps, **kw), pcm, bps))

    for ch in range(1, 9):
        for bps in (4, 8, 12, 16, 20, 24):
            n = int(rng.integers(300, 900))
            pcm = fw.random_pcm(rng, n, ch, bps)
            add(f'ch{ch}-bps{bps}', pcm, bps, blocksize=192 if ch > 4 else 256,
                sub=_kinds(('verbatim', 'fixed', 'lpc', 'fixed'), (0, 1, 2, 3, 4, 8), part_order=2,
                           method_cycle=(0, 1), esc_cycle=((), (1,), (0, 2))))
    for assign in (8, 9, 10):
        for bps in (8, 16, 24):
            pcm = fw.random_pcm(rng, 1500, 2, bps)
            add(f'stereo{assign}-bps{bps}', pcm, bps, blocksize=512, assign=lambda fi, a=assign: a,
                sub=_kinds(('lpc', 'fixed', 'verbatim'), (32, 4, 1), prec=15, part_order=3, method_cycle=(1, 0)))
    pcm = fw.random_pcm(rng, 4000, 2, 16, wasted=3)
    add('wasted-bits', pcm, 16, blocksize=1024, sub=_kinds(('fixed', 'lpc'), (2, 12), wasted=3))
    pcm = np.repeat(rng.integers(-100, 100, size=(5, 1)), 400, axis=0)
    add('constant', pcm, 16, blocksize=400, variable=True, blocks=[400] * 5, sub=_kinds(('constant',), (0,)))
    pcm = fw.random_pcm(rng, 3000, 1, 16)
    add('lpc32-prec15-shift15', pcm, 16, blocksize=1000, variable=True, blocks=[1000, 1000, 1000],
        sub=_kinds(('lpc',), (32,), prec=15, shift=15, part_order=3, method_cycle=(1,)))
    pcm = fw.random_pcm(rng, 2000, 1, 16)
    add('lpc-shift0', pcm, 16, blocksize=500, variable=True, blocks=[500] * 4,
        sub=_kinds(('lpc',), (1, 3), prec=1, shift=0))
    pcm = np.zeros((1000, 1), dtype=np.int64)
    add('escape-0-bits', pcm, 16, blocksize=1000,
        sub=_kinds(('fixed',), (1,), part_order=3, esc_cycle=((0, 1, 2, 3, 4, 5, 6, 7),)))
    pcm = fw.random_pcm(rng, 2500, 1, 16)
    add('variable-blocks', pcm, 16, blocksize=4096, variable=True, blocks=[16, 700, 1000, 17, 767],
        min_bs=16, sub=_kinds(('fixed', 'verbatim'), (2,)))
    pcm = fw.random_pcm(rng, 70000, 1, 12)
    add('block-65535', pcm, 12, blocksize=65535, sub=_kinds(('fixed',), (2,), part_order=0))
    pcm = fw.random_pcm(rng, 700, 1, 8)
    add('block-16', pcm, 8, blocksize=16, sub=_kinds(('fixed', 'verbatim'), (1,)))
    for rate, code in ((22050, 13), (44100, 14), (48000, 12), (8000, 0), (11025, 13), (96000, 11)):
        pcm = fw.random_pcm(rng, 1200, 1, 16)
        add(f'rate{rate}-code{code}', pcm, 16, rate=rate, blocksize=240,
            frame=lambda fi, c=code: dict(rate_code=c, bs_code=6 if fi % 2 else 7, bps_code=0 if fi % 2 else None))
    pcm = fw.random_pcm(rng, 130 * 200, 1, 16)
    add('multibyte-frame-numbers', pcm, 16, blocksize=200, sub=_kinds(('fixed',), (2,)))
    pcm = fw.random_pcm(rng, 3000, 1, 16)
    add('multibyte-sample-numbers', pcm, 16, variable=True, blocks=[150, 2700, 150], min_bs=16,
        sub=_kinds(('fixed',), (2,)))
    add('fake-sync-in-payload', fake_sync_pcm(rng), 8, blocksize=256, sub=lambda fi, c, x: dict(kind='verbatim'))
    return out


def fake_sync_pcm(rng):
    """8-bit mono samples that spell out complete frame headers with a valid CRC-8: in a verbatim frame (a one-byte
    subframe header, one byte per sample) they sit byte aligned in the payload."""
    si = dict(rate=16000, bps=8)
    fake = fake_headers(si)
    blocks = []
    for _ in range(4):
        b = rng.integers(-128, 128, size=256)
        pos = int(rng.integers(0, 256 - len(fake)))
        b[pos:pos + len(fake)] = np.frombuffer(fake, dtype=np.int8)
        blocks.append(b)
    return np.concatenate(blocks)[:, None].astype(np.int64)


def fake_headers(si):
    return fw.frame_header(256, 0, 1, 0, 0, si) + fw.frame_header(256, 512, 2, 0, 0, si)
