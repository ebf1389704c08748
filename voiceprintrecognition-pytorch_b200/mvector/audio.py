"""Minimal AudioSegment: the surface of ``yeaudio.audio.AudioSegment`` that predict.py touches (predict.py:192-211):
``samples`` (float32 mono in [-1, 1]), ``sample_rate``, ``duration``, ``from_file`` / ``from_ndarray`` / ``from_bytes``,
``resample``, ``normalize``, ``vad``.  yeaudio (requirements.txt:12) is a third-party package absent from the reference tree and
from this image; decoding/resampling sit OUTSIDE the parity boundary (SURVEY.md 8a3: parity starts at identical
waveforms).  Decoding covers the uncompressed PCM containers -- WAV (integer, float, A-law and mu-law, also
WAVE_FORMAT_EXTENSIBLE), RF64 / BW64 and AIFF / AIFF-C -- and native FLAC (RFC 9639).  Either segment knows its rate and
duration from the header alone.  A FLAC segment is decoded by vp_flac_decode the first time its samples are read; a PCM
segment's samples are converted by numpy on first read (pcm.to_mono), and both give a device row without a host copy
(``decode_device``: vp_flac_decode / vp_pcm_decode).  Integers become float32 mono with ``pcm_to_mono``; pcm.py states
the rule for floats and G.711.  Other input, and a RIFF file the PCM parser refuses, still goes to the standard
library's ``wave`` reader."""
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
    if isinstance(seg, (FlacSegment, PcmSegment)) and seg._samples is None:
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


class FlacSegment(AudioSegment):
    """A native FLAC stream: ``sample_rate`` and ``duration`` come from STREAMINFO without decoding; ``samples`` are
    decoded on the current CUDA device (vp_flac_decode) the first time they are read, and ``decode_device`` gives them
    as a device row without a host copy.  ``name`` labels the stream in errors."""

    def __init__(self, data, name='<flac>'):
        from .flac import parse_streaminfo
        self.data = bytes(data)
        self.info = parse_streaminfo(self.data)
        self.name = str(name)
        self.sample_rate = self.info.sample_rate
        self._samples = None

    @property
    def samples(self):
        if self._samples is None:
            decode_segments([self])
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
        """The decoded stream as a CUDA float32 row [total_samples] on ``engine``'s device (ValueError when refused);
        the row is kept, so a second call on the same device decodes nothing."""
        row = getattr(self, '_device_row', None)
        if row is None or row.device != engine.device:
            rows, _ = engine.decode_flac([self.data], [self.info], [self.name])
            self._device_row = row = rows[0]
        return row


class PcmSegment(AudioSegment):
    """An uncompressed PCM container file (WAV, RF64 / BW64, AIFF / AIFF-C): ``sample_rate`` and ``duration`` come from
    the header without converting; ``samples`` are converted on the host by numpy (pcm.to_mono) the first time they are
    read, and ``decode_device`` converts the file's bytes on the device (vp_pcm_decode) into the same row.  ``name``
    labels the file in errors."""

    def __init__(self, data, name='<pcm>'):
        from .pcm import parse_header
        self.data = bytes(data)
        self.info = parse_header(self.data)
        self.name = str(name)
        self.sample_rate = self.info.sample_rate
        self._samples = None

    @property
    def samples(self):
        if self._samples is None:
            from .pcm import to_mono
            self._samples = to_mono(self.data, self.info)
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
        """The converted file as a CUDA float32 row [frames] on ``engine``'s device; the row is kept, so a second call on
        the same device converts nothing."""
        row = getattr(self, '_device_row', None)
        if row is None or row.device != engine.device:
            rows, _ = engine.decode_pcm([self.data], [self.info], [self.name])
            self._device_row = row = rows[0]
        return row
