"""Plain Python FLAC decoder written from RFC 9639, the reference the device decoder is tested against: sequential,
frame after frame from the first frame offset, every CRC checked.  Any deviation from the format raises ValueError."""
import numpy as np

from flac_writer import crc8, crc16


class BitReader:
    def __init__(self, data, pos=0):
        self.data, self.bit = data, pos * 8

    def u(self, n):
        v = 0
        for _ in range(n):
            byte = self.bit >> 3
            if byte >= len(self.data):
                raise ValueError('read past the end of the frame')
            v = (v << 1) | ((self.data[byte] >> (7 - (self.bit & 7))) & 1)
            self.bit += 1
        return v

    def s(self, n):
        if n == 0:
            return 0
        v = self.u(n)
        return v - (1 << n) if v >> (n - 1) else v

    def unary(self):
        q = 0
        while self.u(1) == 0:
            q += 1
        return q


def streaminfo(data):
    if data[:4] != b'fLaC':
        raise ValueError('no magic')
    pos, last, info = 4, False, None
    while not last:
        last, t, ln = data[pos] >> 7, data[pos] & 0x7F, int.from_bytes(data[pos + 1:pos + 4], 'big')
        if t == 0:
            b = data[pos + 4:pos + 4 + 34]
            v = int.from_bytes(b[10:18], 'big')
            info = dict(min_bs=int.from_bytes(b[0:2], 'big'), max_bs=int.from_bytes(b[2:4], 'big'), rate=v >> 44,
                        ch=((v >> 41) & 7) + 1, bps=((v >> 36) & 31) + 1, total=v & ((1 << 36) - 1))
        pos += 4 + ln
    info['frame_offset'] = pos
    return info


RATES = [None, 88200, 176400, 192000, 8000, 16000, 22050, 24000, 32000, 44100, 48000, 96000]
BPS = [None, 8, 12, None, 16, 20, 24, None]
FIXED = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


def _header(data, pos, info):
    r = BitReader(data, pos)
    if r.u(15) != 0x7FFC:
        raise ValueError('no sync code')
    variable = r.u(1)
    bsc, rc, chc, bpc = r.u(4), r.u(4), r.u(4), r.u(3)
    if r.u(1):
        raise ValueError('reserved header bit set')
    lead = r.u(8)
    n = 0
    while n < 8 and (lead << n) & 0x80:
        n += 1
    if n == 1 or n > 7 or (n == 7 and not variable):
        raise ValueError('invalid coded number')
    num = lead & (0x7F >> n) if n else lead
    for _ in range(max(n - 1, 0)):
        c = r.u(8)
        if c >> 6 != 2:
            raise ValueError('invalid coded number continuation')
        num = (num << 6) | (c & 0x3F)
    if bsc == 0:
        raise ValueError('reserved block size code')
    bs = {1: 192}.get(bsc) or (576 << (bsc - 2) if bsc <= 5 else None) or (256 << (bsc - 8) if bsc >= 8 else None)
    if bsc == 6:
        bs = r.u(8) + 1
    elif bsc == 7:
        bs = r.u(16) + 1
    if rc == 15:
        raise ValueError('invalid sample rate code')
    rate = info['rate'] if rc == 0 else RATES[rc] if rc < 12 else None
    if rc == 12:
        rate = r.u(8) * 1000
    elif rc == 13:
        rate = r.u(16)
    elif rc == 14:
        rate = r.u(16) * 10
    if chc > 10:
        raise ValueError('reserved channel assignment')
    if bpc in (3, 7):
        raise ValueError('reserved or unsupported bit depth code')
    bps = info['bps'] if bpc == 0 else BPS[bpc]
    end = r.bit // 8
    if r.u(8) != crc8(data[pos:end]):
        raise ValueError('header CRC-8 mismatch')
    start = num if variable else num * info['max_bs']
    if rate != info['rate'] or bps != info['bps'] or (chc + 1 if chc < 8 else 2) != info['ch']:
        raise ValueError('frame header contradicts STREAMINFO')
    return r, bs, chc, bps, start


def _subframe(r, bs, bits):
    if r.u(1):
        raise ValueError('subframe padding bit set')
    t = r.u(6)
    wasted = r.unary() + 1 if r.u(1) else 0
    sb = bits - wasted
    if sb < 1:
        raise ValueError('wasted bits exceed the sample size')
    if t == 0:
        x = [r.s(sb)] * bs
    elif t == 1:
        x = [r.s(sb) for _ in range(bs)]
    elif 8 <= t <= 12 or t >= 32:
        order = t - 8 if t <= 12 else t - 31
        if order > bs:
            raise ValueError('predictor order exceeds the block size')
        x = [r.s(sb) for _ in range(order)]
        if t >= 32:
            prec = r.u(4) + 1
            if prec == 16:
                raise ValueError('invalid LPC precision')
            shift = r.s(5)
            if shift < 0:
                raise ValueError('negative LPC shift')
            coefs = [r.s(prec) for _ in range(order)]
        else:
            coefs, shift = FIXED[order], 0
        method = r.u(2)
        if method > 1:
            raise ValueError('reserved residual coding method')
        pbits = 5 if method else 4
        po = r.u(4)
        psize = bs >> po
        if psize << po != bs or psize < order:
            raise ValueError('invalid partition order')
        res = []
        for p in range(1 << po):
            cnt = psize - order if p == 0 else psize
            k = r.u(pbits)
            if k == (1 << pbits) - 1:
                nb = r.u(5)
                res += [r.s(nb) for _ in range(cnt)]
            else:
                for _ in range(cnt):
                    u = (r.unary() << k) | r.u(k)
                    if u >= 1 << 32:
                        raise ValueError('residual out of range')
                    res.append((u >> 1) ^ -(u & 1))
        for i, e in enumerate(res):
            acc = sum(c * x[order + i - 1 - j] for j, c in enumerate(coefs))
            v = (acc >> shift) + e
            if not -(1 << (sb - 1)) <= v < (1 << (sb - 1)):
                raise ValueError('predicted sample out of range')
            x.append(v)
    else:
        raise ValueError(f'reserved subframe type {t}')
    return [v << wasted for v in x]


def decode(data):
    """FLAC bytes -> (integer PCM [total, ch] int64, STREAMINFO dict)."""
    info = streaminfo(data)
    out = np.zeros((info['total'], info['ch']), dtype=np.int64)
    pos, expect = info['frame_offset'], 0
    while pos < len(data):
        r, bs, chc, bps, start = _header(data, pos, info)
        if start != expect or start + bs > info['total']:
            raise ValueError('frames do not tile the stream')
        chans = []
        for c in range(info['ch']):
            side = (chc == 8 and c == 1) or (chc == 9 and c == 0) or (chc == 10 and c == 1)
            chans.append(_subframe(r, bs, bps + side))
        if r.u(-r.bit % 8):
            raise ValueError('non-zero frame padding')
        end = r.bit // 8
        if end + 2 > len(data) or int.from_bytes(data[end:end + 2], 'big') != crc16(data[pos:end]):
            raise ValueError('frame CRC-16 mismatch')
        if chc >= 8:
            a, b = np.array(chans[0], dtype=np.int64), np.array(chans[1], dtype=np.int64)
            if chc == 8:
                L, R = a, a - b
            elif chc == 9:
                L, R = a + b, b
            else:
                m = (a << 1) | (b & 1)
                L, R = (m + b) >> 1, (m - b) >> 1
            lim = 1 << (bps - 1)
            if (L < -lim).any() or (L >= lim).any() or (R < -lim).any() or (R >= lim).any():
                raise ValueError('decorrelated sample out of range')
            chans = [L, R]
        out[start:start + bs] = np.stack([np.asarray(c, dtype=np.int64) for c in chans], axis=1)
        pos, expect = end + 2, start + bs
    if expect != info['total']:
        raise ValueError('frames do not cover total_samples')
    return out, info
