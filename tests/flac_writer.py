"""Test encoder of native FLAC streams (RFC 9639).  It only has to emit VALID streams, not small ones, so every field
is chosen explicitly -- per frame the blocking strategy, block-size / sample-rate / bit-depth codes and channel
assignment, per subframe the coding, predictor order, LPC precision and shift, wasted bits, residual method, partition
order and escaped partitions.  Any quantised LPC coefficients give a lossless stream."""
import numpy as np

RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10,
              96000: 11}
BPS_CODES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6}
FIXED = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


def crc8(data):
    c = 0
    for b in data:
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
    return c


def crc16(data):
    c = 0
    for b in data:
        c ^= b << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
    return c


class BitWriter:
    def __init__(self):
        self.bits = []

    def u(self, v, n):
        assert 0 <= v < (1 << n) or n == 0, (v, n)
        self.bits.extend((v >> (n - 1 - i)) & 1 for i in range(n))

    def s(self, v, n):
        assert -(1 << (n - 1)) <= v < (1 << (n - 1)), (v, n)
        self.u(v & ((1 << n) - 1), n)

    def unary(self, q):
        self.bits.extend([0] * q + [1])

    def align(self):
        self.bits.extend([0] * (-len(self.bits) % 8))

    def bytes(self):
        assert len(self.bits) % 8 == 0
        a = np.packbits(np.array(self.bits, dtype=np.uint8)) if self.bits else np.zeros(0, np.uint8)
        return a.tobytes()


def coded_number(v):
    if v < 0x80:
        return bytes([v])
    for n in range(2, 8):
        if v < (1 << (5 * n + 1)) or n == 7:
            break
    out = []
    for _ in range(n - 1):
        out.append(0x80 | (v & 0x3F))
        v >>= 6
    lead = (0xFF << (8 - n)) & 0xFF
    return bytes([lead | v] + out[::-1])


def _bits_for(values):
    """Signed bits that hold every value."""
    m = max((int(abs(int(v)) * 2 - (1 if v < 0 else 0)) for v in values), default=0)
    return max(1, int(m).bit_length() + 1) if m else 0


def _rice_param(u, pbits):
    m = int(np.mean(u)) if len(u) else 0
    return min(max(m.bit_length() - 1, 0), (1 << pbits) - 2)


def write_residual(w, res, bs, order, part_order, method, escape_parts=(), params=None):
    pbits = 5 if method else 4
    w.u(method, 2)
    w.u(part_order, 4)
    psize = bs >> part_order
    pos = 0
    for p in range(1 << part_order):
        n = psize - order if p == 0 else psize
        r = [int(x) for x in res[pos:pos + n]]
        pos += n
        u = [(x << 1) if x >= 0 else ((-x) << 1) - 1 for x in r]
        if p in escape_parts:
            nb = _bits_for(r)
            w.u((1 << pbits) - 1, pbits)
            w.u(nb, 5)
            for x in r:
                if nb:
                    w.s(x, nb)
            continue
        k = params[p] if params is not None else _rice_param(u, pbits)
        w.u(k, pbits)
        for x in u:
            w.unary(x >> k)
            w.u(x & ((1 << k) - 1), k)
    assert pos == len(res)


def predict(x, coefs, shift):
    """Residuals of x under the predictor (exact integers)."""
    x = [int(v) for v in x]
    order = len(coefs)
    res = []
    for i in range(order, len(x)):
        acc = sum(c * x[i - 1 - j] for j, c in enumerate(coefs))
        res.append(x[i] - (acc >> shift))
    return res


def write_subframe(w, x, bits, kind='auto', order=2, prec=12, shift=None, wasted=0, part_order=0, method=0,
                   escape_parts=(), coefs=None, rng=None, params=None):
    """One subframe of the integer samples x (``bits`` per sample before the wasted-bits shift)."""
    x = [int(v) for v in x]
    bs = len(x)
    if wasted:
        assert all(v % (1 << wasted) == 0 for v in x)
        x = [v >> wasted for v in x]
    sb = bits - wasted
    w.u(0, 1)
    if kind == 'constant':
        assert len(set(x)) == 1
        w.u(0, 6)
    elif kind == 'verbatim':
        w.u(1, 6)
    elif kind == 'fixed':
        w.u(8 + order, 6)
    elif kind == 'lpc':
        w.u(31 + order, 6)
    else:
        raise ValueError(kind)
    if wasted:
        w.u(1, 1)
        w.unary(wasted - 1)
    else:
        w.u(0, 1)
    if kind == 'constant':
        w.s(x[0], sb)
        return
    if kind == 'verbatim':
        for v in x:
            w.s(v, sb)
        return
    for v in x[:order]:
        w.s(v, sb)
    if kind == 'fixed':
        res = predict(x, FIXED[order], 0)
    else:
        if coefs is None:
            rng = rng or np.random.default_rng(0)
            hi = 1 << (prec - 1)
            lim = max(1, hi // order)                # sum |c| <= 2^(prec-1): |prediction| <= max |x|
            coefs = [int(c) for c in rng.integers(-lim, lim, size=order)]
        shift = prec - 1 if shift is None else shift
        w.u(prec - 1, 4)
        w.s(shift, 5)
        for c in coefs:
            w.s(c, prec)
        res = predict(x, coefs, shift)
    write_residual(w, res, bs, order, part_order, method, escape_parts, params)


def frame_header(bs, start, fn, variable, assign, si, bs_code=None, rate_code=None, bps_code=None):
    """Header bytes (with CRC-8) of one frame: bs_code / rate_code / bps_code None = the natural code."""
    rate, bps = si['rate'], si['bps']
    if bs_code is None:
        table = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, 256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12, 8192: 13,
                 16384: 14, 32768: 15}
        bs_code = table.get(bs, 6 if bs <= 256 else 7)
    if rate_code is None:
        rate_code = RATE_CODES.get(rate, 0)
    if bps_code is None:
        bps_code = BPS_CODES.get(bps, 0)
    h = bytearray([0xFF, 0xF8 | variable, (bs_code << 4) | rate_code, (assign << 4) | (bps_code << 1)])
    h += coded_number(start if variable else fn)
    if bs_code == 6:
        h.append(bs - 1)
    elif bs_code == 7:
        h += (bs - 1).to_bytes(2, 'big')
    if rate_code == 12:
        h.append(rate // 1000)
    elif rate_code == 13:
        h += rate.to_bytes(2, 'big')
    elif rate_code == 14:
        h += (rate // 10).to_bytes(2, 'big')
    h.append(crc8(h))
    return bytes(h)


def channel_ints(pcm, assign):
    """[bs, ch] left/right integers -> per-subframe integer lists and their extra bit (side channel)."""
    if assign < 8:
        return [pcm[:, c] for c in range(pcm.shape[1])], [0] * pcm.shape[1]
    L, R = pcm[:, 0].astype(np.int64), pcm[:, 1].astype(np.int64)
    S = L - R
    if assign == 8:
        return [L, S], [0, 1]
    if assign == 9:
        return [S, R], [1, 0]
    return [(L + R) >> 1, S], [0, 1]


def encode(pcm, rate, bps, blocksize=4096, variable=False, blocks=None, assign=None, sub=None, frame=None,
           min_bs=None, max_bs=None, max_framesize=True, extra_blocks=(), seed=0, frames_out=None):
    """Integer PCM [n, ch] -> FLAC bytes.

    blocks: explicit block sizes (variable blocking, or fixed with a short last block); assign(frame_index) -> channel
    assignment; sub(frame_index, channel, samples) -> write_subframe keyword dict; frame(frame_index) -> frame_header
    keyword dict (codes).  extra_blocks: (type, payload) metadata blocks after STREAMINFO.  frames_out: a list that
    receives each frame's bytes after its header (subframes, padding and CRC-16)."""
    pcm = np.asarray(pcm, dtype=np.int64)
    if pcm.ndim == 1:
        pcm = pcm[:, None]
    n, ch = pcm.shape
    rng = np.random.default_rng(seed)
    if blocks is None:
        blocks = [blocksize] * (n // blocksize) + ([n % blocksize] if n % blocksize else [])
    assert sum(blocks) == n
    si = dict(rate=rate, bps=bps)
    frames, start = [], 0
    for fi, bs in enumerate(blocks):
        a = assign(fi) if assign else (ch - 1)
        hdr = frame_header(bs, start, fi, int(variable), a, si, **(frame(fi) if frame else {}))
        w = BitWriter()
        w.bits.extend(np.unpackbits(np.frombuffer(hdr, dtype=np.uint8)).tolist())
        chans, extra = channel_ints(pcm[start:start + bs], a)
        for c, (x, e) in enumerate(zip(chans, extra)):
            kw = sub(fi, c, x) if sub else {}
            if 'kind' not in kw:
                kw['kind'] = 'fixed'
                kw.setdefault('order', min(2, bs))
            write_subframe(w, x, bps + e, rng=rng, **kw)
        w.align()
        body = w.bytes()
        frames.append(body + crc16(body).to_bytes(2, 'big'))
        if frames_out is not None:
            frames_out.append(frames[-1][len(hdr):])
        start += bs
    if variable:
        body = blocks[:-1] or blocks
        mn = max(16, min(body))
        mx = max(max(blocks), mn)
    else:
        mn = mx = blocksize
    mn = mn if min_bs is None else min_bs
    mx = mx if max_bs is None else max_bs
    fsizes = [len(f) for f in frames]
    si_bytes = _streaminfo(mn, mx, min(fsizes), max(fsizes) if max_framesize else 0, rate, ch, bps, n)
    meta = [(0, si_bytes)] + list(extra_blocks)
    out = bytearray(b'fLaC')
    for i, (t, payload) in enumerate(meta):
        out.append((0x80 if i == len(meta) - 1 else 0) | t)
        out += len(payload).to_bytes(3, 'big')
        out += payload
    return bytes(out) + b''.join(frames)


def _streaminfo(mn, mx, fmin, fmax, rate, ch, bps, total):
    v = (rate << 44) | ((ch - 1) << 41) | ((bps - 1) << 36) | total
    return (mn.to_bytes(2, 'big') + mx.to_bytes(2, 'big') + fmin.to_bytes(3, 'big') + fmax.to_bytes(3, 'big') +
            v.to_bytes(8, 'big') + bytes(16))


def random_pcm(rng, n, ch, bps, wasted=0, smooth=True):
    """Integer PCM [n, ch] in range for bps bits (a smoothed random walk, so predictors have something to predict)."""
    hi = 1 << (bps - 1)
    if smooth:
        x = np.cumsum(rng.integers(-hi // 16 - 1, hi // 16 + 2, size=(n, ch)), axis=0)
        x = (x % (2 * hi)) - hi
    else:
        x = rng.integers(-hi, hi, size=(n, ch))
    if wasted:
        x = (x >> wasted) << wasted
    return np.clip(x, -hi, hi - 1).astype(np.int64)
