"""Uncompressed PCM containers on the host side: the header parser, the numpy conversion and the device conversion of
whole files.

The containers are RIFF/WAVE (format tags PCM, IEEE float, A-law, mu-law and WAVE_FORMAT_EXTENSIBLE with those
sub-formats), RF64 / BW64 with their ds64 chunk, and AIFF / AIFF-C (NONE, twos, sowt, fl32, fl64, ulaw, alaw).  The
parser reads only the headers -- never a sample -- so a segment knows its rate and duration without converting.  The
samples become float32 mono by one rule (include/vpb200.h): integers of container width N as x / 2^(N-1)
(``audio.pcm_to_mono``), float32 as stored, float64 rounded to float32, G.711 through its 16-bit expansion, then
numpy's float32 mean over the channels.  ``to_mono`` applies it with numpy; ``vp_pcm_decode`` (csrc/pcm.cu) applies it
on the device, bit for bit the same, to a ``PcmBatch``: the codec's audio.EncodedBatch, whose per-row table holds each
row's absolute byte offset."""
import struct
from dataclasses import dataclass

import numpy as np

from .audio import EncodedBatch

# VP_PCM_* of include/vpb200.h
U8, S8, S16LE, S16BE, S24LE, S24BE, S32LE, S32BE, F32LE, F32BE, F64LE, F64BE, ULAW, ALAW = range(1, 15)
WIDTH = {U8: 1, S8: 1, S16LE: 2, S16BE: 2, S24LE: 3, S24BE: 3, S32LE: 4, S32BE: 4, F32LE: 4, F32BE: 4, F64LE: 8,
         F64BE: 8, ULAW: 1, ALAW: 1}
MAX_FRAMES = 2 ** 31 - 1
MAX_CHANNELS = 8

_GUID_TAIL = b'\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71'    # KSDATAFORMAT_SUBTYPE_* after the tag
_COMPRESSED = {0x0002: 'Microsoft ADPCM', 0x0011: 'IMA ADPCM', 0x0031: 'GSM 6.10', 0x0050: 'MPEG', 0x0055: 'MPEG Layer 3',
               0x0092: 'Dolby AC-3', 0x1610: 'AAC', 0xF1AC: 'FLAC'}


@dataclass(frozen=True)
class PcmInfo:
    sample_rate: int
    channels: int
    format: int                # one of the VP_PCM_* codes above
    frames: int                # samples per channel
    data_offset: int           # byte offset of the first sample in the file

    @property
    def width(self):
        return WIDTH[self.format]

    @property
    def duration(self):
        return self.frames / float(self.sample_rate)


def is_pcm(head):
    """True when the bytes start like a container this module parses (RIFF, RF64, BW64 or an IFF FORM)."""
    return bytes(head[:4]) in (b'RIFF', b'RF64', b'BW64', b'FORM')


def parse_header(data):
    """Headers of a WAV / RF64 / BW64 / AIFF / AIFF-C file (bytes-like) -> PcmInfo.  Never reads sample data.

    A data chunk larger than the bytes present, or sized 0 / 0xFFFFFFFF by a streaming writer, is clamped to the bytes
    present, rounded down to whole frames; a WAV data size of 0 counts as a streaming writer's only when the RIFF size
    is unset too (0 / 0xFFFFFFFF) or ends at the data chunk, else the data chunk is empty.  Raises ValueError for a malformed or truncated header and
    NotImplementedError, naming the reason, for what is not uncompressed PCM of 8 / 16 / 24 / 32-bit integers or
    32 / 64-bit floats in 1 to 8 channels."""
    d = memoryview(data)
    magic = bytes(d[:4])
    if magic in (b'RIFF', b'RF64', b'BW64'):
        return _parse_riff(d, magic)
    if magic == b'FORM':
        return _parse_aiff(d)
    raise ValueError('not a WAV / RF64 / AIFF file: no RIFF, RF64, BW64 or FORM magic')


def _chunks(d, pos, endian):
    """(id, body offset, declared size) of each chunk header from ``pos`` on; a chunk body is padded to even length."""
    fmt = '<I' if endian == 'little' else '>I'
    while pos + 8 <= len(d):
        cid, size = bytes(d[pos:pos + 4]), struct.unpack_from(fmt, d, pos + 4)[0]
        yield cid, pos + 8, size
        pos += 8 + size + (size & 1)


def _clamp(d, body, size, frame_bytes, streaming=True):
    """Whole frames of a sample chunk at ``body`` declaring ``size`` bytes, clamped to the bytes present.  A size of
    0xFFFFFFFF, or of 0 when the container says it was never finalised (``streaming``), runs to the end of the file."""
    avail = max(len(d) - body, 0)
    if size == 0xFFFFFFFF or (size == 0 and streaming) or size > avail:
        size = avail
    return size // frame_bytes


def _finish(rate, channels, fmt, frames, offset):
    if not 0 < rate < 2 ** 31:
        raise ValueError(f'sample rate {rate}: outside 1 .. 2^31 - 1')
    if frames > MAX_FRAMES:
        raise NotImplementedError(f'{frames} samples per channel: not supported (at most 2^31 - 1)')
    return PcmInfo(sample_rate=int(rate), channels=int(channels), format=fmt, frames=int(frames), data_offset=int(offset))


def _check_channels(ch):
    if ch < 1:
        raise ValueError(f'{ch} channels')
    if ch > MAX_CHANNELS:
        raise NotImplementedError(f'{ch} channels: not supported (1 to {MAX_CHANNELS})')


def _int_format(bits, little, unsigned8):
    width = (bits + 7) // 8
    if bits < 1 or width not in (1, 2, 3, 4):
        raise NotImplementedError(f'{bits}-bit integer samples: not supported (8, 16, 24 or 32-bit containers)')
    if width == 1:
        return U8 if unsigned8 else S8
    return {2: (S16BE, S16LE), 3: (S24BE, S24LE), 4: (S32BE, S32LE)}[width][little]


def _float_format(bits, little):
    if bits not in (32, 64):
        raise NotImplementedError(f'{bits}-bit float samples: not supported (32 or 64)')
    return {32: (F32BE, F32LE), 64: (F64BE, F64LE)}[bits][little]


def _wav_format(tag, bits):
    if tag == 1:
        return _int_format(bits, True, True)
    if tag == 3:
        return _float_format(bits, True)
    if tag in (6, 7):
        if bits != 8:
            raise NotImplementedError(f"{bits}-bit {'A-law' if tag == 6 else 'mu-law'}: not supported (8 bits)")
        return ALAW if tag == 6 else ULAW
    name = _COMPRESSED.get(tag, 'compressed or unknown')
    raise NotImplementedError(f'WAV format tag 0x{tag:04x} ({name}): not supported (uncompressed PCM, float, A-law or '
                              f'mu-law only)')


def _parse_riff(d, magic):
    if len(d) < 12:
        raise ValueError(f'truncated {magic.decode()} header')
    if bytes(d[8:12]) != b'WAVE':
        raise ValueError(f'{magic.decode()} file of form {bytes(d[8:12])!r}, not WAVE')
    fmt = data = ds64_size = None
    for cid, body, size in _chunks(d, 12, 'little'):
        if cid == b'ds64' and magic != b'RIFF':
            if size < 24 or body + 24 > len(d):
                raise ValueError('truncated ds64 chunk')
            ds64_size = struct.unpack_from('<Q', d, body + 8)[0]
        elif cid == b'fmt ':
            if size < 16 or body + 16 > len(d):
                raise ValueError('truncated fmt chunk')
            tag, ch, rate, _, align, bits = struct.unpack_from('<HHIIHH', d, body)
            if tag == 0xFFFE:
                if size < 40 or body + 40 > len(d):
                    raise ValueError('truncated WAVE_FORMAT_EXTENSIBLE fmt chunk')
                guid = bytes(d[body + 24:body + 40])
                if guid[2:] != _GUID_TAIL:
                    raise NotImplementedError(f'WAVE_FORMAT_EXTENSIBLE sub-format GUID {guid.hex()}: not supported')
                tag = struct.unpack_from('<H', guid)[0]
            fmt = (tag, ch, rate, align, bits)
        elif cid == b'data':
            if size == 0xFFFFFFFF and ds64_size is not None:
                size = ds64_size                       # RF64: the 64-bit size is in ds64
            data = (body, size)
            if fmt is not None:
                break
    if fmt is None:
        raise ValueError('WAV file has no fmt chunk')
    if data is None:
        raise ValueError('WAV file has no data chunk')
    tag, ch, rate, align, bits = fmt
    # a data size of 0 means "not finalised" only when the RIFF size is unset too (0 or 0xFFFFFFFF) or ends at the data
    # chunk's header; otherwise the data chunk is empty and any bytes after it belong to later chunks
    riff_size = struct.unpack_from('<I', d, 4)[0]
    streaming = riff_size in (0, 0xFFFFFFFF) or 8 + riff_size <= data[0]
    _check_channels(ch)
    f = _wav_format(tag, bits)                    # the valid-bits field of an EXTENSIBLE header is not read: the
    if align != ch * WIDTH[f]:                    # container width scales the samples
        raise ValueError(f'block align {align} contradicts {ch} channels of {WIDTH[f]} bytes')
    return _finish(rate, ch, f, _clamp(d, data[0], data[1], align, streaming), data[0])


def _ext80(b):
    """An IEEE 754 80-bit extended float (AIFF's sample rate) -> int; NotImplementedError when it is not an integer."""
    sign, exp, mant = b[0] >> 7, ((b[0] & 0x7F) << 8) | b[1], int.from_bytes(b[2:10], 'big')
    if sign or mant == 0 or exp == 0x7FFF:
        raise ValueError('AIFF sample rate is not a positive finite number')
    e = exp - 16383 - 63
    if e >= 0:
        return mant << min(e, 64)
    if mant & ((1 << -e) - 1):
        raise NotImplementedError(f'non-integer AIFF sample rate {mant / 2.0 ** -e}: not supported')
    return mant >> -e


_AIFC = {b'NONE': 'twos', b'twos': 'twos', b'sowt': 'sowt', b'fl32': F32BE, b'FL32': F32BE, b'fl64': F64BE,
         b'FL64': F64BE, b'ulaw': ULAW, b'ULAW': ULAW, b'alaw': ALAW, b'ALAW': ALAW}


def _parse_aiff(d):
    if len(d) < 12:
        raise ValueError('truncated FORM header')
    form = bytes(d[8:12])
    if form not in (b'AIFF', b'AIFC'):
        raise ValueError(f'FORM file of type {form!r}, not AIFF or AIFF-C')
    comm = ssnd = None
    for cid, body, size in _chunks(d, 12, 'big'):
        if cid == b'COMM':
            need = 22 if form == b'AIFC' else 18
            if size < need or body + need > len(d):
                raise ValueError('truncated COMM chunk')
            ch, frames, bits = struct.unpack_from('>hIh', d, body)
            comm = (ch, frames, bits, bytes(d[body + 8:body + 18]), bytes(d[body + 18:body + 22]) if form == b'AIFC'
                    else b'NONE')
        elif cid == b'SSND':
            if body + 8 > len(d):
                raise ValueError('truncated SSND chunk')
            offset = struct.unpack_from('>I', d, body)[0]          # the samples start offset bytes into the block
            streaming = size in (0, 0xFFFFFFFF) or size < 8 + offset
            ssnd = (body + 8 + offset, 0 if streaming else size - 8 - offset)
        if comm is not None and ssnd is not None:
            break
    if comm is None:
        raise ValueError('AIFF file has no COMM chunk')
    if ssnd is None:
        raise ValueError('AIFF file has no SSND chunk')
    ch, frames, bits, rate80, comp = comm
    _check_channels(ch)
    kind = _AIFC.get(comp)
    if kind is None:
        raise NotImplementedError(f'AIFF-C compression {comp!r}: not supported (NONE, twos, sowt, fl32, fl64, ulaw, '
                                  f'alaw)')
    f = _int_format(bits, kind == 'sowt', False) if isinstance(kind, str) else kind
    rate = _ext80(rate80)
    body, size = ssnd
    return _finish(rate, ch, f, min(frames, _clamp(d, body, size, ch * WIDTH[f])), body)


# ------------------------------------------------------------------------------------------------ conversion
def _g711_tables():
    """int16 expansions of all 256 mu-law and A-law bytes (ITU-T G.711), the twin of csrc/pcm.cu."""
    u = ~np.arange(256) & 0xFF
    t = ((((u & 0x0F) << 3) + 0x84) << ((u >> 4) & 7)) - 0x84
    mu = np.where(u & 0x80, -t, t)
    a = np.arange(256) ^ 0x55
    seg = (a >> 4) & 7
    m = (a & 0x0F) << 4
    t = np.where(seg == 0, m + 8, (m + 0x108) << np.maximum(seg - 1, 0))
    al = np.where(a & 0x80, t, -t)
    return mu.astype(np.int16), al.astype(np.int16)


_ULAW, _ALAW = _g711_tables()


def to_mono(data, info):
    """The samples of a parsed file (bytes-like ``data``, its PcmInfo) -> float32 mono, by numpy.  vp_pcm_decode gives
    the same row bit for bit."""
    from .audio import pcm_to_mono
    f, ch = info.format, info.channels
    raw = np.frombuffer(data, dtype=np.uint8, count=info.frames * ch * info.width, offset=info.data_offset)
    if f == U8:
        return pcm_to_mono(raw.astype(np.int16) - 128, ch, 8)
    if f == S8:
        return pcm_to_mono(raw.view(np.int8), ch, 8)
    if f in (ULAW, ALAW):
        return pcm_to_mono((_ULAW if f == ULAW else _ALAW)[raw], ch, 16)
    if f in (S24LE, S24BE):
        b = raw.reshape(-1, 3).astype(np.int32)
        if f == S24BE:
            b = b[:, ::-1]
        return pcm_to_mono((b[:, 0] << 8 | b[:, 1] << 16 | b[:, 2] << 24) >> 8, ch, 24)
    dt = {S16LE: '<i2', S16BE: '>i2', S32LE: '<i4', S32BE: '>i4', F32LE: '<f4', F32BE: '>f4', F64LE: '<f8',
          F64BE: '>f8'}[f]
    x = raw.view(dt)
    if f in (S16LE, S16BE, S32LE, S32BE):
        return pcm_to_mono(x, ch, 8 * info.width)
    x = x.astype(np.float32)
    return x.reshape(-1, ch).mean(axis=1) if ch > 1 else x


# ------------------------------------------------------------------------------------------------ device conversion
def _info_struct(info, base):
    from ._lib import PcmInfo as CInfo
    return CInfo(base + info.data_offset, info.frames, info.channels, info.format, 0, 0)


class PcmBatch(EncodedBatch):
    """Device inputs of one vp_pcm_decode over several files: their concatenated bytes and a vp_pcm_info per row, which
    holds the row's absolute byte offset, so ``rows(lo, hi)`` is a batch over the same bytes that uploads nothing."""
    label, unit = 'PCM', 'row'

    @staticmethod
    def _length(si):
        return si.frames

    def _tables(self, device):
        import torch
        raw = b''.join(bytes(_info_struct(si, int(o))) for si, o in zip(self.infos, self.offsets[:-1]))
        self.info = torch.frombuffer(bytearray(raw or b'\0'), dtype=torch.uint8).pin_memory().to(device,
                                                                                                 non_blocking=True)

    def rows(self, lo, hi, stream=None):
        """The batch of rows lo..hi: a slice of the info table over the same bytes (``stream`` is unused)."""
        v = PcmBatch.__new__(PcmBatch)
        v.infos, v.names, v.nbytes, v.lengths, v.data = self.infos[lo:hi], self.names[lo:hi], self.nbytes, \
            self.lengths[lo:hi], self.data
        size = self.info.numel() // max(len(self), 1)
        v.info = self.info[lo * size:hi * size]
        return v

    def decode_into(self, engine, out, ld, status, stream=None):
        engine.decode_pcm_into(self, out, ld, status, stream)

    def host_row(self, i, engine):
        """Row i converted by numpy: the same row as the device's."""
        return to_mono(self.file(i), self.infos[i])
