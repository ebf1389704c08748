"""Test writer of uncompressed PCM containers: RIFF/WAVE (plain and WAVE_FORMAT_EXTENSIBLE), RF64 / BW64 and AIFF /
AIFF-C, with every header field given explicitly so the tests can also write what a correct writer would not (a wrong
block align, a streaming data size, odd chunks before the samples).  Sample encoding is by the format names of
pcm_oracle (``'s24le'``, ``'f64be'``, ``'ulaw'``, ...)."""
import struct

import numpy as np

import pcm_oracle as po

WAV_TAG = {'u8': 1, 's16le': 1, 's24le': 1, 's32le': 1, 'f32le': 3, 'f64le': 3, 'alaw': 6, 'ulaw': 7}
AIFC_TYPE = {'s8': b'twos', 's16be': b'NONE', 's24be': b'twos', 's32be': b'NONE', 'f32be': b'fl32', 'f64be': b'FL64',
             'ulaw': b'ulaw', 'alaw': b'ALAW'}
SOWT = ('s16le', 's24le', 's32le')


def random_samples(rng, fmt, n):
    """n stored values of format ``fmt`` spanning its whole range: ints at both extremes, floats in [-1.5, 1.5] with
    exact zeros and +-1, G.711 every byte."""
    if fmt in ('ulaw', 'alaw', 'u8', 's8'):
        v = rng.integers(0, 256, size=n)
        v[:min(n, 256)] = np.arange(min(n, 256))
        return v if fmt != 's8' else v - 128
    if fmt[0] == 's':
        bits = int(fmt[1:3])
        v = rng.integers(-2 ** (bits - 1), 2 ** (bits - 1), size=n)
        v[:2] = [-2 ** (bits - 1), 2 ** (bits - 1) - 1][:min(n, 2)]
        return v
    v = rng.uniform(-1.5, 1.5, size=n)
    v[:4] = [0.0, 1.0, -1.0, 1e-30][:min(n, 4)]
    return v


def encode(values, fmt):
    """Stored bytes of ``values`` (interleaved) in format ``fmt``."""
    v = np.asarray(values)
    if fmt in ('ulaw', 'alaw', 'u8'):
        return v.astype(np.uint8).tobytes()
    if fmt == 's8':
        return v.astype(np.int8).tobytes()
    if fmt in ('s24le', 's24be'):
        b = (v.astype(np.int64) & 0xFFFFFF).astype(np.uint32)
        cols = [b & 0xFF, (b >> 8) & 0xFF, b >> 16]
        if fmt == 's24be':
            cols = cols[::-1]
        return np.stack(cols, axis=1).astype(np.uint8).tobytes()
    end = '<' if fmt.endswith('le') else '>'
    kind = 'i' if fmt[0] == 's' else 'f'
    return v.astype(f'{end}{kind}{int(fmt[1:3]) // 8}').tobytes()


def chunk(cid, body, endian='<'):
    """A chunk: id, size, body and the pad byte of an odd-sized body."""
    return cid + struct.pack(endian + 'I', len(body)) + body + (b'\0' if len(body) & 1 else b'')


def guid(tag):
    return struct.pack('<H', tag) + b'\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71'


def wav(samples, rate, ch, fmt, *, tag=None, bits=None, block_align=None, extensible=False, valid_bits=None,
        sub_guid=None, before=(), after=(), data_size=None, magic=b'RIFF', riff_size=None, ds64_data=None,
        fmt_first=True):
    """A WAV file of the stored bytes ``samples``.  ``before`` / ``after``: extra (id, body) chunks around data;
    ``data_size`` overrides the data chunk's size field; magic RF64 / BW64 writes a ds64 chunk first holding
    ``ds64_data`` (default: the true size) and 0xFFFFFFFF in the RIFF and data size fields."""
    width = po.WIDTH[fmt]
    tag = WAV_TAG[fmt] if tag is None else tag
    bits = 8 * width if bits is None else bits
    block_align = ch * width if block_align is None else block_align
    head = struct.pack('<HHIIHH', 0xFFFE if extensible else tag, ch, rate, rate * block_align, block_align, bits)
    if extensible:
        head += struct.pack('<HHI', 22, bits if valid_bits is None else valid_bits, (1 << ch) - 1)
        head += guid(tag) if sub_guid is None else sub_guid
    elif tag != 1:
        head += struct.pack('<H', 0)
    chunks = []
    if magic != b'RIFF':
        size = len(samples) if ds64_data is None else ds64_data
        chunks.append(chunk(b'ds64', struct.pack('<QQQI', 0, size, size // block_align, 0)))
        data_size = 0xFFFFFFFF if data_size is None else data_size
    fmt_chunk = chunk(b'fmt ', head)
    if fmt_first:
        chunks.append(fmt_chunk)
    chunks += [chunk(cid, body) for cid, body in before]
    size = len(samples) if data_size is None else data_size
    chunks.append(b'data' + struct.pack('<I', size) + samples + (b'\0' if len(samples) & 1 and after else b''))
    if not fmt_first:
        chunks.append(fmt_chunk)
    chunks += [chunk(cid, body) for cid, body in after]
    body = b'WAVE' + b''.join(chunks)
    rs = (0xFFFFFFFF if magic != b'RIFF' else len(body)) if riff_size is None else riff_size
    return magic + struct.pack('<I', rs) + body


def ext80(value):
    """IEEE 754 80-bit extended encoding of a positive number (an AIFF sample rate)."""
    if isinstance(value, int):
        e = value.bit_length() - 1
        mant = value << (63 - e)
    else:
        m, e = np.frexp(value)
        e -= 1
        mant = int(m * 2 ** 64)
    return struct.pack('>HQ', e + 16383, mant)


def aiff(samples, rate, ch, frames, fmt, *, comp=None, bits=None, rate80=None, ssnd_offset=0, before=(),
         ssnd_size=None, aifc=None):
    """An AIFF (``comp`` None and a big-endian integer ``fmt``) or AIFF-C file of the stored bytes ``samples``.
    ``comp`` defaults to AIFC_TYPE[fmt] ('sowt' for little-endian integers)."""
    width = po.WIDTH[fmt]
    if comp is None and (aifc or fmt not in ('s8', 's16be', 's24be', 's32be')):
        comp = b'sowt' if fmt in SOWT else AIFC_TYPE[fmt]
    bits = (16 if fmt in ('ulaw', 'alaw') else 8 * width) if bits is None else bits
    comm = struct.pack('>hIh', ch, frames, bits) + (ext80(rate) if rate80 is None else rate80)
    if comp is not None:
        comm += comp + b'\x04none\x00'             # pascal string, padded to even
    ssnd = struct.pack('>II', ssnd_offset, 0) + b'\xAB' * ssnd_offset + samples
    chunks = [chunk(b'COMM', comm, '>')] + [chunk(cid, body, '>') for cid, body in before]
    size = len(ssnd) if ssnd_size is None else ssnd_size
    chunks.append(b'SSND' + struct.pack('>I', size) + ssnd + (b'\0' if len(ssnd) & 1 else b''))
    body = (b'AIFC' if comp is not None else b'AIFF') + b''.join(chunks)
    return b'FORM' + struct.pack('>I', len(body)) + body


WAV_FORMATS = ('u8', 's16le', 's24le', 's32le', 'f32le', 'f64le', 'ulaw', 'alaw')
AIFF_FORMATS = ('s8', 's16be', 's24be', 's32be', 's16le', 's24le', 's32le', 'f32be', 'f64be', 'ulaw', 'alaw')


def matrix(rng, frames=(37, 64, 5)):
    """Every format in every container it can take, 1 to 8 channels: [(name, file bytes, format, channels, stored
    values, rate)].  Frame counts cycle through ``frames`` (odd counts leave odd-sized data chunks)."""
    out = []
    k = 0
    for container in ('wav', 'extensible', 'rf64', 'bw64', 'aiff'):
        for fmt in (WAV_FORMATS if container != 'aiff' else AIFF_FORMATS):
            for ch in range(1, 9):
                n = frames[k % len(frames)]
                k += 1
                rate = (8000, 16000, 22050, 44100, 48000)[k % 5]
                vals = random_samples(rng, fmt, n * ch)
                raw = encode(vals, fmt)
                if container == 'aiff':
                    data = aiff(raw, rate, ch, n, fmt, aifc=(k % 2 == 0), ssnd_offset=k % 3)
                elif container in ('rf64', 'bw64'):
                    data = wav(raw, rate, ch, fmt, magic=container.upper().encode())
                else:
                    data = wav(raw, rate, ch, fmt, extensible=container == 'extensible',
                               before=[(b'LIST', b'INFOx' * (k % 3))] if k % 2 else ())
                out.append((f'{container}-{fmt}-{ch}ch', data, fmt, ch, vals, rate))
    return out
