"""FLAC (RFC 9639) on the host side: the metadata parser and the device decode of whole streams.

The host reads only the ``fLaC`` magic and the metadata blocks -- STREAMINFO gives the rate, channel count, bit depth
and length, so a segment's duration is known without decoding.  The frames are decoded on the device by
``vp_flac_decode`` (csrc/flac.cu); there is no host decoder behind it.  ``FlacBatch`` is the codec's audio.EncodedBatch:
the per-stream tables vp_flac_decode reads and the rebased batch of a staging stage's rows."""
from dataclasses import dataclass

import numpy as np

from .audio import EncodedBatch

MAGIC = b'fLaC'


@dataclass(frozen=True)
class StreamInfo:
    sample_rate: int
    channels: int
    bps: int
    total_samples: int
    min_blocksize: int
    max_blocksize: int
    min_framesize: int
    max_framesize: int
    frame_offset: int          # byte offset of the first frame: the byte after the last metadata block

    @property
    def duration(self):
        return self.total_samples / float(self.sample_rate)


def is_flac(head):
    """True when the bytes start like a native FLAC stream -- or like the wrapped forms (Ogg, an ID3 tag) that
    parse_streaminfo refuses by name."""
    head = bytes(head[:4])
    return head == MAGIC or head == b'OggS' or head[:3] == b'ID3'


def parse_streaminfo(data):
    """Metadata of a native FLAC stream (bytes-like) -> StreamInfo.  Never reads frame data.

    Raises ValueError for a truncated or malformed header and NotImplementedError, naming the reason, for what the
    decoder does not take: Ogg-encapsulated or ID3-tagged streams, an unknown sample count and 32-bit samples."""
    data = memoryview(data)
    head = bytes(data[:4])
    if head[:3] == b'ID3':
        raise NotImplementedError('ID3-tagged stream: not supported (native FLAC or PCM WAV only)')
    if head == b'OggS':
        raise NotImplementedError('Ogg-encapsulated stream (Ogg FLAC): not supported (native FLAC or PCM WAV only)')
    if head != MAGIC:
        raise ValueError('not a FLAC stream: no fLaC magic')
    pos, info, last = 4, None, False
    while not last:
        if pos + 4 > len(data):
            raise ValueError('truncated FLAC metadata block header')
        h = bytes(data[pos:pos + 4])
        last, btype, length = bool(h[0] & 0x80), h[0] & 0x7F, int.from_bytes(h[1:4], 'big')
        pos += 4
        if pos + length > len(data):
            raise ValueError(f'truncated FLAC metadata block (type {btype}, {length} bytes)')
        if btype == 127:
            raise ValueError('invalid FLAC metadata block type 127')
        if info is None:
            if btype != 0 or length != 34:
                raise ValueError('the first FLAC metadata block is not a 34-byte STREAMINFO')
            info = _streaminfo(bytes(data[pos:pos + 34]))
        elif btype == 0:
            raise ValueError('second STREAMINFO block')
        pos += length
    if pos >= len(data):
        raise ValueError('FLAC stream has no frames')
    return StreamInfo(frame_offset=pos, **info)


def _streaminfo(b):
    v = int.from_bytes(b[10:18], 'big')
    info = dict(min_blocksize=int.from_bytes(b[0:2], 'big'), max_blocksize=int.from_bytes(b[2:4], 'big'),
                min_framesize=int.from_bytes(b[4:7], 'big'), max_framesize=int.from_bytes(b[7:10], 'big'),
                sample_rate=v >> 44, channels=((v >> 41) & 7) + 1, bps=((v >> 36) & 31) + 1,
                total_samples=v & ((1 << 36) - 1))
    if info['min_blocksize'] < 16 or info['max_blocksize'] < info['min_blocksize']:
        raise ValueError(f"invalid FLAC block sizes {info['min_blocksize']}..{info['max_blocksize']}")
    if info['sample_rate'] == 0:
        raise ValueError('FLAC sample rate 0')
    if info['bps'] < 4:
        raise ValueError(f"invalid FLAC bit depth {info['bps']}")
    if info['bps'] > 24:
        raise NotImplementedError(f"{info['bps']}-bit FLAC: not supported (4 to 24 bits)")
    if info['total_samples'] == 0:
        raise NotImplementedError('FLAC stream of unknown length (total samples 0): not supported')
    return info


def _info_struct(si):
    from ._lib import FlacInfo
    return FlacInfo(si.total_samples, si.sample_rate, si.channels, si.bps, si.min_blocksize, si.max_blocksize,
                    si.min_framesize, si.max_framesize, 0)


class FlacBatch(EncodedBatch):
    """Device inputs of one vp_flac_decode over several streams: the concatenated bytes and the per-stream tables
    (``offsets`` and ``frame_off`` as vp_flac_decode's stream and first-frame offsets, a vp_flac_info per stream)."""
    label, unit = 'FLAC', 'stream'

    @staticmethod
    def _length(si):
        return si.total_samples

    def _tables(self, device):
        import torch
        self.frame_off = self.offsets[:-1] + np.array([si.frame_offset for si in self.infos], dtype=np.int64)
        self.max_frames = int(sum(-(-si.total_samples // si.min_blocksize) for si in self.infos))
        raw = b''.join(bytes(_info_struct(si)) for si in self.infos)
        self.info = torch.frombuffer(bytearray(raw or b'\0'), dtype=torch.uint8).to(device)
        self.stream_off_dev = torch.from_numpy(self.offsets).to(device)
        self.frame_off_dev = torch.from_numpy(self.frame_off).to(device)

    def rows(self, lo, hi, stream):
        """The batch of rows lo..hi: the bytes stay where they are, the tables are rebased onto row lo and uploaded on
        ``stream``.  The scan and link passes walk every byte from ``data`` on, so a stage passes only its own bytes."""
        import torch
        v = FlacBatch.__new__(FlacBatch)
        base = int(self.offsets[lo])
        v.infos, v.names = self.infos[lo:hi], self.names[lo:hi]
        v.offsets, v.frame_off = self.offsets[lo:hi + 1] - base, self.frame_off[lo:hi] - base
        v.nbytes = int(v.offsets[-1])
        v.max_frames = int(sum(-(-si.total_samples // si.min_blocksize) for si in v.infos))
        v.lengths = self.lengths[lo:hi]
        v.data = self.data[base:]
        v.info = self.info[lo * (self.info.numel() // len(self)):]
        with torch.cuda.stream(stream):
            v.stream_off_dev = torch.from_numpy(v.offsets).to(self.data.device, non_blocking=True)
            v.frame_off_dev = torch.from_numpy(v.frame_off).to(self.data.device, non_blocking=True)
        return v

    def decode_into(self, engine, out, ld, status, stream=None):
        engine.decode_flac_into(self, out, ld, status, stream)

    def host_row(self, i, engine):
        """Stream i decoded on ``engine``'s device and copied to the host."""
        rows, _ = engine.decode_flac([self.file(i)], [self.infos[i]], [self.names[i]])
        return rows[0].cpu().numpy()
