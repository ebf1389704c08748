"""Minimal AudioSegment: the surface of ``yeaudio.audio.AudioSegment`` that predict.py touches (predict.py:192-211):
``samples`` (float32 mono in [-1, 1]), ``sample_rate``, ``duration``, ``from_file`` / ``from_ndarray`` / ``from_bytes``,
``resample``, ``normalize``, ``vad``.  yeaudio (requirements.txt:12) is a third-party package absent from the reference tree and
from this image; decoding/resampling sit OUTSIDE the parity boundary (SURVEY.md 8a3: parity starts at identical
waveforms).  Decoding covers PCM WAV via the standard library only."""
import io
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
            pcm = np.frombuffer(raw, dtype='<i2').astype(np.float32) / 32768.0
        elif sw == 4:
            pcm = np.frombuffer(raw, dtype='<i4').astype(np.float32) / 2147483648.0
        elif sw == 1:
            pcm = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
        else:
            raise ValueError(f'unsupported WAV sample width {sw}')
        if ch > 1:
            pcm = pcm.reshape(-1, ch).mean(axis=1)
        return cls(pcm, sr)

    @classmethod
    def from_file(cls, file):
        return cls._from_wave(file)

    @classmethod
    def from_bytes(cls, data):
        return cls._from_wave(io.BytesIO(data))

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

    def vad(self, return_seconds=False, frame_ms=30.0, rel_threshold_db=-35.0, min_speech_ms=250.0, min_silence_ms=300.0):
        """Voice-activity segments ``[{'start': ..., 'end': ...}, ...]`` in samples (or seconds).

        Stand-in for yeaudio's model-based ``AudioSegment.vad`` (absent third-party code, outside the parity boundary):
        frame RMS energy against a threshold ``rel_threshold_db`` below the loudest frame, silences shorter than
        ``min_silence_ms`` bridged, bursts shorter than ``min_speech_ms`` dropped.  Same return format, so
        ``SpeakerDiarization.segments_audio`` (infer_utils/speaker_diarization.py) consumes either."""
        sr = self.sample_rate
        hop = max(1, int(sr * frame_ms / 1000.0))
        n = self.samples.shape[0]
        if n < hop:
            return []
        nf = n // hop
        x = self.samples[:nf * hop].astype(np.float64).reshape(nf, hop)
        db = 10.0 * np.log10(np.maximum((x * x).mean(axis=1), 1e-12))
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
