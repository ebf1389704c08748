"""FLAC (RFC 9639) on the host side: the metadata parser and the device decode of whole streams.

The host reads only the ``fLaC`` magic and the metadata blocks -- STREAMINFO gives the rate, channel count, bit depth
and length, so a segment's duration is known without decoding.  The frames are decoded on the device by
``vp_flac_decode`` (csrc/flac.cu); there is no host decoder behind it."""
from dataclasses import dataclass

import numpy as np

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


class FlacBatch:
    """Device inputs of one vp_flac_decode over several streams: the concatenated bytes and the per-stream tables.
    ``names`` label the items in errors."""

    def __init__(self, streams, infos, device, names=None, stream=None):
        """The bytes go up in one pinned copy on ``stream`` (default: the current stream)."""
        import torch
        if stream is not None:
            with torch.cuda.stream(stream):
                self.__init__(streams, infos, device, names)
            return
        self.infos = list(infos)
        self.names = list(names) if names is not None else [f'item {i}' for i in range(len(self.infos))]
        sizes = np.array([len(s) for s in streams], dtype=np.int64)
        self.stream_off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        self.frame_off = self.stream_off[:-1] + np.array([si.frame_offset for si in self.infos], dtype=np.int64)
        self.nbytes = int(self.stream_off[-1])
        self.max_frames = int(sum(-(-si.total_samples // si.min_blocksize) for si in self.infos))
        self.lengths = np.array([si.total_samples for si in self.infos], dtype=np.int64)
        host = torch.empty(max(self.nbytes, 1), dtype=torch.uint8, pin_memory=True)
        hv = host.numpy()
        for o, s in zip(self.stream_off[:-1], streams):
            hv[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
        self.data = host.to(device, non_blocking=True)
        raw = b''.join(bytes(_info_struct(si)) for si in self.infos)
        self.info = torch.frombuffer(bytearray(raw or b'\0'), dtype=torch.uint8).to(device)
        self.stream_off_dev = torch.from_numpy(self.stream_off).to(device)
        self.frame_off_dev = torch.from_numpy(self.frame_off).to(device)
        self._host = host            # the pinned source stays alive until the copy has run
        self._src = [memoryview(hv[o:o + len(s)]) for o, s in zip(self.stream_off[:-1], streams)]

    def __len__(self):
        return len(self.infos)


def check_status(status, names):
    """Raise ValueError naming every refused item of a decode (status: host int32 array)."""
    bad = np.flatnonzero(np.asarray(status))
    if bad.size:
        items = ', '.join(f'{names[i]} (status {int(status[i])})' for i in bad[:8])
        raise ValueError(f'FLAC decode refused {bad.size} stream(s): {items}')


class DeviceFlacRows:
    """Rows of ``_embed_waves`` decoded from FLAC streams on the device: row i is stream i at its native rate, ``lens[i]``
    samples zero filled to the slot's width.  The compressed bytes of every row go up in one pinned copy on the copy
    stream; a staging slot is then written by vp_flac_decode of its rows instead of the host gather and H2D copy.
    ``check`` raises ValueError naming a refused stream (after the caller's result copy)."""

    def __init__(self, engine, segs, copy_stream):
        import torch
        self.engine, self.stream = engine, copy_stream
        self.infos = [s.info for s in segs]
        self.names = [s.name for s in segs]
        self.lens = np.array([si.total_samples for si in self.infos], dtype=np.int32)
        self.batch = FlacBatch([s.data for s in segs], self.infos, engine.device, self.names, stream=copy_stream)
        with torch.cuda.stream(copy_stream):
            self.status = torch.zeros(len(segs), dtype=torch.int32, device=engine.device)

    def __len__(self):
        return len(self.infos)

    def _stage(self, lo, hi):
        """A FlacBatch view of rows lo..hi: the bytes stay where they are, the tables are rebased onto row lo."""
        import torch
        b = self.batch
        v = FlacBatch.__new__(FlacBatch)
        base = int(b.stream_off[lo])
        v.infos, v.names = b.infos[lo:hi], b.names[lo:hi]
        v.stream_off, v.frame_off = b.stream_off[lo:hi + 1] - base, b.frame_off[lo:hi] - base
        v.nbytes = int(v.stream_off[-1])
        v.max_frames = int(sum(-(-si.total_samples // si.min_blocksize) for si in v.infos))
        v.lengths = b.lengths[lo:hi]
        v.data = b.data[base:]
        v.info = b.info[lo * (b.info.numel() // len(b)):]
        with torch.cuda.stream(self.stream):
            v.stream_off_dev = torch.from_numpy(v.stream_off).to(self.engine.device, non_blocking=True)
            v.frame_off_dev = torch.from_numpy(v.frame_off).to(self.engine.device, non_blocking=True)
        return v

    def gather(self, lo, hi, dst, ld, stream):
        """Rows lo..hi decoded into the device slot ``dst`` [hi - lo, ld] on ``stream``."""
        self.engine.decode_flac_into(self._stage(lo, hi), dst, ld, self.status[lo:hi], stream)

    def __getitem__(self, i):
        """Host copy of row i (ConditionPlan.check recomputes a flagged row's gain from it)."""
        rows, _ = self.engine.decode_flac([bytes(self.batch._src[i])], [self.infos[i]], [self.names[i]])
        return rows[0].cpu().numpy()

    def check(self):
        check_status(self.status.cpu().numpy(), self.names)
