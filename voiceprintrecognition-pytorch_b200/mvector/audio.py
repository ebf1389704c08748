"""Minimal AudioSegment: the surface of ``yeaudio.audio.AudioSegment`` that predict.py touches (predict.py:192-211):
``samples`` (float32 mono in [-1, 1]), ``sample_rate``, ``duration``, ``from_file`` / ``from_ndarray`` / ``from_bytes``,
``resample``, ``normalize``, ``vad``.  yeaudio (requirements.txt:12) is a third-party package absent from the reference tree and
from this image; decoding/resampling sit OUTSIDE the parity boundary (SURVEY.md 8a3: parity starts at identical
waveforms).  Decoding covers the uncompressed PCM containers -- WAV (integer, float, A-law and mu-law, also
WAVE_FORMAT_EXTENSIBLE), RF64 / BW64 and AIFF / AIFF-C -- and native FLAC (RFC 9639).  Both are EncodedSegments: a
file kept as its bytes, whose rate and duration come from the header alone.  A FLAC segment is decoded by vp_flac_decode
the first time its samples are read; a PCM segment's samples are converted by numpy on first read (pcm.to_mono), and
both give a device row without a host copy (``decode_device``).  On the device an encoded file goes through one path
whatever its codec: an EncodedBatch uploads the files' bytes in one pinned copy, the codec's subclass (flac.FlacBatch,
pcm.PcmBatch) adds its tables and its decode, and DeviceEncodedRows writes the staging rows of ``_embed_waves`` from it.
Integers become float32 mono with ``pcm_to_mono``; pcm.py states the rule for floats and G.711.  Other input, and a
RIFF file the PCM parser refuses, still goes to the standard library's ``wave`` reader."""
import io
import os
import wave
from math import gcd

import numpy as np


def resample_ratio(sample_rate, target_rate):
    """(up, down) of ``AudioSegment.resample`` from ``sample_rate`` to ``target_rate``: the rates divided by their gcd."""
    g = gcd(int(target_rate), int(sample_rate))
    return int(target_rate) // g, int(sample_rate) // g


def resampled_length(n, up, down):
    """Samples resample_poly returns for n input samples: ceil(n * up / down), in int64 (ten minutes at 44.1 kHz times
    up = 160 does not fit in int32).  Works elementwise on arrays."""
    return -(-np.asarray(n, dtype=np.int64) * np.asarray(up, dtype=np.int64) // np.asarray(down, dtype=np.int64))


def polyphase_taps(up, down):
    """resample_poly's anti-aliasing filter for (up, down), laid out per phase for the device resampler
    (include/vpb200.h, vp_resample) -> (table float64 [up * nt], nt, n_pre_remove).

    scipy's recipe: max_rate = max(up, down), half_len = 10 max_rate, h = firwin(2 half_len + 1, 1 / max_rate,
    window=('kaiser', 5.0)) * up, n_pre_pad = down - half_len % down, n_pre_remove = (half_len + n_pre_pad) // down.
    hpad = (n_pre_pad zeros, h); table[p * nt + m] = hpad[p + m * up], zero past the end of hpad."""
    from scipy.signal import firwin
    max_rate = max(up, down)
    half_len = 10 * max_rate
    h = firwin(2 * half_len + 1, 1.0 / max_rate, window=('kaiser', 5.0)) * up
    n_pre_pad = down - half_len % down
    hpad = np.concatenate([np.zeros(n_pre_pad), h])
    nt = -(-len(hpad) // up)
    flat = np.zeros(up * nt)
    flat[:len(hpad)] = hpad
    return np.ascontiguousarray(flat.reshape(nt, up).T).reshape(-1), nt, (half_len + n_pre_pad) // down


def pcm_to_mono(ints, channels, bps):
    """Interleaved integer PCM -> float32 mono: x / 2^(bps - 1) in float32, then (channels > 1) numpy's float32 mean over
    each sample's channels.  vp_flac_decode reproduces this bit for bit (include/vpb200.h)."""
    x = np.asarray(ints).astype(np.float32) / np.float32(2 ** (bps - 1))
    if channels > 1:
        x = x.reshape(-1, channels).mean(axis=1)
    return x


_engines = {}


def _engine(device=None):
    """The Engine FLAC segments decode with: one per CUDA device (default: the current one)."""
    import torch
    from .engine import Engine
    idx = torch.cuda.current_device() if device is None else torch.device(device).index
    if idx not in _engines:
        _engines[idx] = Engine(idx)
    return _engines[idx]


def device_samples(seg, engine):
    """A segment's samples as a CUDA float32 row on ``engine``'s device: an undecoded FLAC or PCM segment is converted
    there from its file's bytes and its samples never visit the host; any other segment's samples are uploaded."""
    import torch
    if isinstance(seg, EncodedSegment) and seg._samples is None:
        return seg.decode_device(engine)
    return torch.from_numpy(np.ascontiguousarray(seg.samples, dtype=np.float32)).to(engine.device)


def decode_segments(segs, engine=None):
    """Give every undecoded FlacSegment of ``segs`` its host samples with ONE device decode (ValueError names a
    refused item)."""
    todo = [s for s in segs if isinstance(s, FlacSegment) and s._samples is None]
    if not todo:
        return
    eng = engine or _engine()
    rows, _ = eng.decode_flac([s.data for s in todo], [s.info for s in todo], [s.name for s in todo])
    host = rows.cpu().numpy()
    for s, r in zip(todo, host):
        s._samples = np.ascontiguousarray(r[:s.info.total_samples])


class AudioSegment:
    def __init__(self, samples, sample_rate):
        s = np.asarray(samples)
        if s.dtype.kind in 'iu':
            s = s.astype(np.float32) / float(2 ** (8 * s.dtype.itemsize - 1))
        s = s.astype(np.float32, copy=False)
        if s.ndim == 2:                       # [n, channels] -> mono
            s = s.mean(axis=1)
        self.samples = s
        self.sample_rate = int(sample_rate)

    @property
    def duration(self):
        return self.samples.shape[0] / float(self.sample_rate)

    @classmethod
    def from_ndarray(cls, data, sample_rate=16000):
        return cls(data, sample_rate)

    @classmethod
    def _from_wave(cls, f):
        with wave.open(f, 'rb') as w:
            n, ch, sw, sr = w.getnframes(), w.getnchannels(), w.getsampwidth(), w.getframerate()
            raw = w.readframes(n)
        if sw == 2:
            ints = np.frombuffer(raw, dtype='<i2')
        elif sw == 4:
            ints = np.frombuffer(raw, dtype='<i4')
        elif sw == 1:
            ints = np.frombuffer(raw, dtype=np.uint8).astype(np.int16) - 128
        else:
            raise ValueError(f'unsupported WAV sample width {sw}')
        return cls(pcm_to_mono(ints, ch, 8 * sw), sr)

    @classmethod
    def from_file(cls, file):
        """A PCM container or native FLAC file (path or binary file object), told apart by its magic; anything else is
        read by ``wave``."""
        from .flac import is_flac
        from .pcm import is_pcm
        if isinstance(file, (str, os.PathLike)):
            with open(file, 'rb') as f:
                head = f.read(4)
                if not (is_flac(head) or is_pcm(head)):
                    return cls._from_wave(file)
                f.seek(0)
                return cls._from_data(f.read(), os.fspath(file))
        return cls._from_data(file.read(), getattr(file, 'name', '<file>'))

    @classmethod
    def from_bytes(cls, data):
        return cls._from_data(data, '<bytes>')

    @classmethod
    def _from_data(cls, data, name):
        from .flac import is_flac
        from .pcm import is_pcm
        if is_flac(data):
            return FlacSegment(data, name=name)
        if is_pcm(data):
            return cls._from_pcm(data, name)
        return cls._from_wave(io.BytesIO(data))

    @classmethod
    def _from_pcm(cls, data, name):
        """A PcmSegment; or, for a RIFF file the PCM parser refuses but the ``wave`` reader reads (integer PCM of more
        than 8 channels, a block align that contradicts the format), the segment the ``wave`` reader gives, as it did
        before the parser existed.  When neither reads the file, the parser's error is raised."""
        try:
            return PcmSegment(data, name=name)
        except (ValueError, NotImplementedError) as err:
            if bytes(data[:4]) != b'RIFF':
                raise
            try:
                return AudioSegment._from_wave(io.BytesIO(data))
            except Exception:  # noqa: BLE001  (the wave reader's own error says less than the parser's)
                raise err from None

    def resample(self, target_sample_rate):
        if target_sample_rate == self.sample_rate:
            return
        from scipy.signal import resample_poly
        g = gcd(int(target_sample_rate), self.sample_rate)
        self.samples = resample_poly(self.samples.astype(np.float64), int(target_sample_rate) // g,
                                     self.sample_rate // g).astype(np.float32)
        self.sample_rate = int(target_sample_rate)

    @property
    def rms_db(self):
        return 10.0 * np.log10(np.mean(self.samples.astype(np.float64) ** 2))

    def normalize(self, target_db=-20, max_gain_db=300.0):
        gain = target_db - self.rms_db
        if gain > max_gain_db:
            raise ValueError(f'cannot normalise to {target_db} dB: gain {gain} dB exceeds {max_gain_db} dB')
        self.samples = (self.samples * (10.0 ** (gain / 20.0))).astype(np.float32)

    @staticmethod
    def vad_hop(sample_rate, frame_ms=30.0):
        """Samples per VAD frame at ``sample_rate``."""
        return max(1, int(sample_rate * frame_ms / 1000.0))

    def frame_energy(self, frame_ms=30.0):
        """Mean square of every whole VAD frame (float64 [n // hop]); ``Engine.frame_energy`` is its device twin."""
        hop = self.vad_hop(self.sample_rate, frame_ms)
        nf = self.samples.shape[0] // hop
        x = self.samples[:nf * hop].astype(np.float64).reshape(nf, hop)
        return (x * x).mean(axis=1)

    def vad(self, return_seconds=False, frame_ms=30.0, rel_threshold_db=-35.0, min_speech_ms=250.0, min_silence_ms=300.0):
        """Voice-activity segments ``[{'start': ..., 'end': ...}, ...]`` in samples (or seconds).

        Stand-in for yeaudio's model-based ``AudioSegment.vad`` (absent third-party code, outside the parity boundary):
        frame RMS energy against a threshold ``rel_threshold_db`` below the loudest frame, silences shorter than
        ``min_silence_ms`` bridged, bursts shorter than ``min_speech_ms`` dropped.  Same return format, so
        ``SpeakerDiarization.segments_audio`` (infer_utils/speaker_diarization.py) consumes either."""
        return self.vad_from_energy(self.frame_energy(frame_ms), self.samples.shape[0], self.sample_rate, return_seconds,
                                    frame_ms, rel_threshold_db, min_speech_ms, min_silence_ms)

    @classmethod
    def vad_from_energy(cls, ms, n, sr, return_seconds=False, frame_ms=30.0, rel_threshold_db=-35.0, min_speech_ms=250.0,
                        min_silence_ms=300.0):
        """The decision half of ``vad``: ``ms`` the frame energies (``frame_energy``) of a recording of ``n`` samples at
        ``sr`` Hz -> the same segments."""
        hop = cls.vad_hop(sr, frame_ms)
        if n < hop:
            return []
        db = 10.0 * np.log10(np.maximum(np.asarray(ms, dtype=np.float64), 1e-12))
        active = db > (db.max() + rel_threshold_db)
        # runs of active frames
        edges = np.flatnonzero(np.diff(np.concatenate([[0], active.astype(np.int8), [0]])))
        runs = [[int(a), int(b)] for a, b in zip(edges[0::2], edges[1::2])]
        merged = []
        gap = int(round(min_silence_ms / frame_ms))
        for r in runs:
            if merged and r[0] - merged[-1][1] < gap:
                merged[-1][1] = r[1]
            else:
                merged.append(r)
        keep = int(round(min_speech_ms / frame_ms))
        out = []
        for a, b in merged:
            if b - a < keep:
                continue
            st, ed = a * hop, min(b * hop, n)
            out.append({'start': st / sr, 'end': ed / sr} if return_seconds else {'start': st, 'end': ed})
        return out


class EncodedSegment(AudioSegment):
    """An encoded audio file kept as its bytes: ``sample_rate`` and ``duration`` come from the header (``info``) without
    decoding; ``samples`` are converted on the host the first time they are read (``_convert``), and ``decode_device``
    gives them as a device row without a host copy.  ``name`` labels the file in errors.  A subclass names its header
    parser, its host conversion and its ``batch_type`` (an EncodedBatch subclass holding the codec's device decode)."""

    def __init__(self, data, name, parse, batch_type):
        self.data = bytes(data)
        self.info = parse(self.data)
        self.name = str(name)
        self.batch_type = batch_type
        self.sample_rate = self.info.sample_rate
        self._samples = None

    @property
    def samples(self):
        if self._samples is None:
            self._samples = self._convert()
        return self._samples

    @samples.setter
    def samples(self, value):
        self._samples = value

    @property
    def duration(self):
        if self._samples is None:
            return self.info.duration
        return self._samples.shape[0] / float(self.sample_rate)

    def decode_device(self, engine):
        """The decoded file as a CUDA float32 row on ``engine``'s device (ValueError when refused); the row is kept, so
        a second call on the same device decodes nothing."""
        row = getattr(self, '_device_row', None)
        if row is None or row.device != engine.device:
            rows, _ = engine.decode_batch(self.batch_type([self.data], [self.info], engine.device, [self.name]))
            self._device_row = row = rows[0]
        return row


class FlacSegment(EncodedSegment):
    """A native FLAC stream (``info``: its flac.StreamInfo).  There is no host decoder: ``samples`` are decoded on the
    current CUDA device (vp_flac_decode) by ``decode_segments``."""

    def __init__(self, data, name='<flac>'):
        from .flac import FlacBatch, parse_streaminfo
        super().__init__(data, name, parse_streaminfo, FlacBatch)

    def _convert(self):
        decode_segments([self])
        return self._samples


class PcmSegment(EncodedSegment):
    """An uncompressed PCM container file (WAV, RF64 / BW64, AIFF / AIFF-C; ``info``: its pcm.PcmInfo): ``samples`` are
    converted on the host by numpy (pcm.to_mono), the same row vp_pcm_decode gives on the device."""

    def __init__(self, data, name='<pcm>'):
        from .pcm import PcmBatch, parse_header
        super().__init__(data, name, parse_header, PcmBatch)

    def _convert(self):
        from .pcm import to_mono
        return to_mono(self.data, self.info)


class EncodedBatch:
    """Device inputs of one decode over several encoded files: their bytes concatenated in ``data`` (file i from
    ``offsets[i]``, ``nbytes`` in all) and each file's decoded length in ``lengths``.  ``names`` label the items in errors.
    A subclass adds its codec's per-row tables (``_tables``), the batch of rows lo..hi a stage decodes
    (``rows(lo, hi, stream)``), the engine's decode (``decode_into``), a row decoded for the host (``host_row``), and the
    ``label`` and ``unit`` its errors name."""

    def __init__(self, files, infos, device, names=None, stream=None):
        """The bytes go up in one pinned copy, then the tables, on ``stream`` (default: the current stream)."""
        import torch
        self.infos = list(infos)
        self.names = list(names) if names is not None else [f'item {i}' for i in range(len(self.infos))]
        self.lengths = np.array([self._length(si) for si in self.infos], dtype=np.int64)
        sizes = np.array([len(f) for f in files], dtype=np.int64)
        self.offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        self.nbytes = int(self.offsets[-1])
        with torch.cuda.stream(stream):
            host = torch.empty(max(self.nbytes, 1), dtype=torch.uint8, pin_memory=True)
            hv = host.numpy()
            for o, f in zip(self.offsets[:-1], files):
                hv[o:o + len(f)] = np.frombuffer(f, dtype=np.uint8)
            self.data = host.to(device, non_blocking=True)
            self._tables(device)
        self._host = host            # the pinned source stays alive until the copy has run

    def __len__(self):
        return len(self.infos)

    def file(self, i):
        """The bytes of file i, read back from the pinned source."""
        return bytes(self._host.numpy()[self.offsets[i]:self.offsets[i + 1]])


def check_status(status, names, label, unit):
    """Raise ValueError naming every refused item of a ``label`` decode (status: host int32 array, one per ``unit``)."""
    bad = np.flatnonzero(np.asarray(status))
    if bad.size:
        items = ', '.join(f'{names[i]} (status {int(status[i])})' for i in bad[:8])
        raise ValueError(f'{label} decode refused {bad.size} {unit}(s): {items}')


class DeviceEncodedRows:
    """Rows of ``_embed_waves`` decoded on the device from EncodedSegments of one class: row i is file i at its native
    rate, ``lens[i]`` samples zero filled to the slot's width.  The files' bytes go up in one pinned copy on the copy
    stream; a staging slot is then written by the device decode of its rows instead of the host gather and H2D copy.
    ``check`` raises ValueError naming a refused file (after the caller's result copy)."""

    def __init__(self, engine, segs, copy_stream):
        import torch
        self.engine, self.stream = engine, copy_stream
        self.batch = segs[0].batch_type([s.data for s in segs], [s.info for s in segs], engine.device,
                                        [s.name for s in segs], copy_stream)
        self.lens = np.array(self.batch.lengths.tolist(), dtype=np.int32)    # a length past int32 raises, never wraps
        with torch.cuda.stream(copy_stream):
            self.status = torch.zeros(len(segs), dtype=torch.int32, device=engine.device)

    def __len__(self):
        return len(self.batch)

    def gather(self, lo, hi, dst, ld, stream):
        """Rows lo..hi decoded into the device slot ``dst`` [hi - lo, ld] on ``stream``."""
        self.batch.rows(lo, hi, self.stream).decode_into(self.engine, dst, ld, self.status[lo:hi], stream)

    def __getitem__(self, i):
        """Host copy of row i (ConditionPlan.check recomputes a flagged row's gain from it)."""
        return self.batch.host_row(i, self.engine)

    def check(self):
        check_status(self.status.cpu().numpy(), self.batch.names, self.batch.label, self.batch.unit)
