"""Independent decoder of stored PCM samples for the tests: bytes of one format -> float32 mono, written from the
conversion rule (include/vpb200.h) and the G.711 standard, without mvector.pcm.

G.711 is expanded from its fields.  mu-law: the byte is complemented; bit 7 is the sign (set = negative), bits 4-6 the
segment e, bits 0-3 the mantissa m; the 14-bit magnitude is (2m + 33) 2^e - 33, times 4 for 16 bits.  A-law: the byte is
XORed with 0x55; bit 7 set = positive; the 13-bit magnitude is 2m + 1 in segment 0 and (2m + 33) 2^(e-1) above, times
8 for 16 bits.  The channel mean is spelled out in numpy's float32 order: the sum starts at +0.0, left to right below 8
values, pairwise ((c0+c1)+(c2+c3))+((c4+c5)+(c6+c7)) for 8, then one division by the count."""
import numpy as np

WIDTH = {'u8': 1, 's8': 1, 'ulaw': 1, 'alaw': 1, 's16le': 2, 's16be': 2, 's24le': 3, 's24be': 3, 's32le': 4,
         's32be': 4, 'f32le': 4, 'f32be': 4, 'f64le': 8, 'f64be': 8}


def ulaw_to_int(byte):
    c = ~int(byte) & 0xFF
    sign, e, m = c >> 7, (c >> 4) & 7, c & 15
    mag = ((2 * m + 33) * 2 ** e - 33) * 4
    return -mag if sign else mag


def alaw_to_int(byte):
    c = int(byte) ^ 0x55
    sign, e, m = c >> 7, (c >> 4) & 7, c & 15
    mag = (2 * m + 1 if e == 0 else (2 * m + 33) * 2 ** (e - 1)) * 8
    return mag if sign else -mag


def values(raw, fmt):
    """Stored bytes -> the float32 value of every sample (interleaved)."""
    b = np.frombuffer(bytes(raw), dtype=np.uint8)
    w = WIDTH[fmt]
    if fmt in ('ulaw', 'alaw'):
        f = ulaw_to_int if fmt == 'ulaw' else alaw_to_int
        ints = np.array([f(x) for x in range(256)], dtype=np.int64)[b]
        return ints.astype(np.float32) / np.float32(2 ** 15)
    if fmt == 'u8':
        return (b.astype(np.int64) - 128).astype(np.float32) / np.float32(128)
    groups = b.reshape(-1, w).astype(np.uint64)
    if fmt.endswith('le') or fmt == 's8':
        groups = groups[:, ::-1]                       # most significant byte first
    u = np.zeros(groups.shape[0], dtype=np.uint64)
    for k in range(w):
        u = (u << np.uint64(8)) | groups[:, k]
    if fmt[0] == 'f':
        if w == 4:
            return u.astype(np.uint32).view(np.float32)
        return u.view(np.float64).astype(np.float32)
    bits = 8 * w
    signed = u.astype(np.int64) - ((u >> np.uint64(bits - 1)) << np.uint64(bits)).astype(np.int64)
    return signed.astype(np.float32) / np.float32(2 ** (bits - 1))


def mean_channels(x, ch):
    """numpy's float32 mean over each frame's ``ch`` values, in its order."""
    f = x.reshape(-1, ch)
    if ch == 1:
        return f[:, 0].copy()
    if ch == 8:
        p = [f[:, 2 * i] + f[:, 2 * i + 1] for i in range(4)]
        s = np.float32(0) + ((p[0] + p[1]) + (p[2] + p[3]))
    else:
        s = np.zeros(f.shape[0], dtype=np.float32)
        for c in range(ch):
            s = s + f[:, c]
    return s / np.float32(ch)


def decode(raw, fmt, ch):
    """Stored bytes of ``fmt`` with ``ch`` interleaved channels -> float32 mono."""
    return mean_channels(values(raw, fmt), ch)
