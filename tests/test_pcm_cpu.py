"""Uncompressed PCM containers on the host (mvector/pcm.py, audio.PcmSegment), no GPU: the header parser over every
format x container x 1-8 channels, odd chunks, RF64 / BW64, clamped data and every refusal; segments that know their
rate and duration without converting; and the numpy conversion against the independent decoder of the tests
(pcm_oracle.py) and, for the WAVs the standard library writes, against the ``wave`` reader it replaces."""
import ctypes
import io
import mmap
import os
import re
import struct
import wave

import numpy as np
import pytest

import pcm_oracle as po
import pcm_writer as pw

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CODE = {'u8': 1, 's8': 2, 's16le': 3, 's16be': 4, 's24le': 5, 's24be': 6, 's32le': 7, 's32be': 8, 'f32le': 9,
        'f32be': 10, 'f64le': 11, 'f64be': 12, 'ulaw': 13, 'alaw': 14}


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.int32)


@pytest.fixture(scope='module')
def cases():
    return pw.matrix(np.random.default_rng(7))


def test_format_codes_follow_the_header():
    from mvector import _lib, pcm
    src = open(os.path.join(ROOT, 'include', 'vpb200.h')).read()
    header = {m.group(1).lower(): int(m.group(2)) for m in re.finditer(r'VP_PCM_(\w+) = (\d+)', src)}
    assert header == CODE
    assert all(getattr(pcm, k.upper()) == v for k, v in CODE.items())
    body = re.search(r'typedef struct vp_pcm_info \{(.*?)\} vp_pcm_info;', src, re.S).group(1)
    fields = [re.match(r'\s*(\w+)\s+(\w+)', d).groups() for d in re.sub(r'/\*.*?\*/', '', body, flags=re.S).split(';')
              if d.strip()]
    ctype = {'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64}
    assert [(n, ctype[t]) for t, n in fields] == list(_lib.PcmInfo._fields_)


def test_matrix_headers(cases):
    from mvector.pcm import parse_header
    assert len(cases) == 8 * 8 * 4 + 11 * 8
    for name, data, fmt, ch, vals, rate in cases:
        info = parse_header(data)
        n = len(vals) // ch
        assert (info.sample_rate, info.channels, info.format, info.frames) == (rate, ch, CODE[fmt], n), name
        assert info.data_offset + n * ch * po.WIDTH[fmt] <= len(data), name
        assert info.duration == n / rate


def test_matrix_samples_equal_the_oracle(cases):
    from mvector.audio import AudioSegment, PcmSegment
    for name, data, fmt, ch, vals, rate in cases:
        seg = AudioSegment.from_bytes(data)
        assert isinstance(seg, PcmSegment), name
        ref = po.decode(pw.encode(vals, fmt), fmt, ch)
        assert seg.samples.dtype == np.float32 and np.array_equal(_bits(seg.samples), _bits(ref)), name


def test_oracle_mean_is_numpys_mean():
    rng = np.random.default_rng(3)
    for ch in range(1, 9):
        x = (rng.standard_normal(4000 * ch) * 10.0 ** rng.integers(-6, 6, 4000 * ch)).astype(np.float32)
        x[:ch] = -0.0
        assert np.array_equal(_bits(po.mean_channels(x, ch)), _bits(x.reshape(-1, ch).mean(axis=1) if ch > 1 else x))


def test_g711_extremes_and_tables():
    from mvector import pcm
    mu = [po.ulaw_to_int(b) for b in range(256)]
    al = [po.alaw_to_int(b) for b in range(256)]
    assert (min(mu), max(mu)) == (-32124, 32124) and (min(al), max(al)) == (-32256, 32256)
    assert po.ulaw_to_int(0xFF) == 0 and po.ulaw_to_int(0x7F) == 0 and po.alaw_to_int(0xD5) == 8
    assert list(pcm._ULAW) == mu and list(pcm._ALAW) == al


@pytest.mark.parametrize('comp,fmt', [(b'NONE', 's16be'), (b'twos', 's24be'), (b'sowt', 's16le'), (b'fl32', 'f32be'),
                                      (b'FL32', 'f32be'), (b'fl64', 'f64be'), (b'FL64', 'f64be'), (b'ulaw', 'ulaw'),
                                      (b'ULAW', 'ulaw'), (b'alaw', 'alaw'), (b'ALAW', 'alaw')])
def test_aifc_compression_names(comp, fmt):
    from mvector.pcm import parse_header, to_mono
    vals = pw.random_samples(np.random.default_rng(1), fmt, 2 * 50)
    data = pw.aiff(pw.encode(vals, fmt), 11025, 2, 50, fmt, comp=comp)
    info = parse_header(data)
    assert (info.format, info.frames, info.sample_rate) == (CODE[fmt], 50, 11025)
    assert np.array_equal(_bits(to_mono(data, info)), _bits(po.decode(pw.encode(vals, fmt), fmt, 2)))


def test_odd_chunks_before_and_after_data():
    from mvector.audio import AudioSegment
    vals = pw.random_samples(np.random.default_rng(2), 'u8', 33)
    raw = pw.encode(vals, 'u8')
    data = pw.wav(raw, 8000, 1, 'u8', before=[(b'LIST', b'INFOISFT\x03\x00\x00\x00ab\x00'), (b'fact', b'\x21\0\0\0'),
                                              (b'junk', b'xyz')], after=[(b'LIST', b'abc')])
    seg = AudioSegment.from_bytes(data)
    assert seg.info.frames == 33 and np.array_equal(seg.samples, po.decode(raw, 'u8', 1))
    later_fmt = pw.wav(raw, 8000, 1, 'u8', fmt_first=False, after=[(b'LIST', b'abc')])   # fmt after an odd data chunk
    assert np.array_equal(AudioSegment.from_bytes(later_fmt).samples, seg.samples)
    aif = pw.aiff(pw.encode(vals - 128, 's8'), 8000, 1, 33, 's8',
                  before=[(b'NAME', b'odd'), (b'ANNO', b'')], ssnd_offset=3)
    assert np.array_equal(AudioSegment.from_bytes(aif).samples, seg.samples)      # u8 - 128 == s8


@pytest.mark.parametrize('magic', [b'RF64', b'BW64'])
def test_rf64_sizes_come_from_ds64(magic):
    from mvector.pcm import parse_header, to_mono
    vals = pw.random_samples(np.random.default_rng(4), 's24le', 2 * 101)
    raw = pw.encode(vals, 's24le')
    data = pw.wav(raw, 48000, 2, 's24le', magic=magic, after=[(b'LIST', b'tail')])
    info = parse_header(data)
    assert info.frames == 101 and np.array_equal(to_mono(data, info), po.decode(raw, 's24le', 2))
    short = pw.wav(raw, 48000, 2, 's24le', magic=magic, ds64_data=6 * 40, after=[(b'LIST', b'tail')])
    assert parse_header(short).frames == 40


def test_data_sizes_clamped_to_the_bytes_present():
    from mvector.pcm import parse_header
    raw = pw.encode(pw.random_samples(np.random.default_rng(5), 's16le', 3 * 20), 's16le')
    # a streaming writer: data size 0 / 0xFFFFFFFF with the RIFF size unset or ending at the data chunk's header (36:
    # 'WAVE', a 16-byte fmt chunk and the data header)
    for size, riff in ((0, 0), (0, 0xFFFFFFFF), (0, 36), (0xFFFFFFFF, None), (0xFFFFFFFF, 0xFFFFFFFF),
                       (len(raw) + 1000, None)):
        assert parse_header(pw.wav(raw, 16000, 3, 's16le', data_size=size, riff_size=riff)).frames == 20, (size, riff)
    assert parse_header(pw.wav(raw, 16000, 3, 's16le')[:-7]).frames == 18          # a partial last frame is dropped
    assert parse_header(pw.wav(raw, 16000, 3, 's16le', data_size=6 * 5)).frames == 5
    aif = pw.aiff(raw, 16000, 3, 20, 's16le', ssnd_size=0xFFFFFFFF)
    assert parse_header(aif).frames == 20
    assert parse_header(aif[:-6]).frames == 19
    assert parse_header(pw.aiff(raw, 16000, 3, 7, 's16le')).frames == 7               # COMM's count wins when smaller


def test_empty_data_chunk_in_a_finalised_file():
    """A data size of 0 in a file whose RIFF size covers later chunks is an empty data chunk, as the wave reader has
    it: the chunks after it are not read as samples."""
    from mvector.pcm import parse_header
    raw = pw.encode(pw.random_samples(np.random.default_rng(6), 's16le', 50), 's16le')
    empty = pw.wav(b'', 16000, 1, 's16le', after=[(b'LIST', b'INFOISFT' + b'x' * 120)])
    assert parse_header(empty).frames == 0
    covered = pw.wav(raw, 16000, 1, 's16le', data_size=0)          # RIFF size patched, data size not
    assert parse_header(covered).frames == 0
    with wave.open(io.BytesIO(empty)) as w:
        assert w.getnframes() == 0


def _wav_fmt_only(tag, bits=16, ch=1, align=None):
    return pw.wav(b'\0' * 64, 16000, ch, 's16le', tag=tag, bits=bits, block_align=align)


@pytest.mark.parametrize('data,exc,msg', [
    (b'RIFF\x10\0\0\0WA', ValueError, 'truncated RIFF header'),
    (b'RIFF\x10\0\0\0AVI LIST', ValueError, 'not WAVE'),
    (b'RIFF\x0c\0\0\0WAVEdata\0\0\0\0', ValueError, 'no fmt chunk'),
    (b'RIFF\x10\0\0\0WAVEfmt \x10\0\0\0\x01\0', ValueError, 'truncated fmt chunk'),
    (pw.wav(b'\0' * 8, 8000, 1, 's16le')[:36], ValueError, 'no data chunk'),
    (_wav_fmt_only(1, 16, 2, align=2), ValueError, 'block align 2 contradicts 2 channels'),
    (_wav_fmt_only(2), NotImplementedError, r'0x0002 \(Microsoft ADPCM\)'),
    (_wav_fmt_only(0x31), NotImplementedError, r'GSM 6\.10'),
    (_wav_fmt_only(0x55), NotImplementedError, 'MPEG Layer 3'),
    (pw.wav(b'\0' * 8, 8000, 1, 's16le', extensible=True, sub_guid=b'\x01' * 16), NotImplementedError,
     'sub-format GUID'),
    (pw.wav(b'\0' * 10, 8000, 1, 's16le', bits=40, block_align=5), NotImplementedError, '40-bit integer'),
    (pw.wav(b'\0' * 8, 8000, 1, 'f32le', bits=16, block_align=2), NotImplementedError, '16-bit float'),
    (pw.wav(b'\0' * 8, 8000, 1, 'ulaw', bits=16, block_align=2), NotImplementedError, '16-bit mu-law'),
    (pw.wav(b'\0' * 18, 8000, 9, 's16le'), NotImplementedError, '9 channels'),
    (pw.wav(b'\0' * 18, 8000, 0, 's16le', block_align=0), ValueError, '0 channels'),
    (pw.wav(b'\0' * 8, 0, 1, 's16le'), ValueError, 'sample rate 0'),
    (b'RF64\xff\xff\xff\xffWAVEds64\x1c\0\0\0' + b'\0' * 8, ValueError, 'truncated ds64'),
    (b'FORM\x04\0\0\0AIFF', ValueError, 'no COMM chunk'),
    (b'FORM\x04\0\0\0AIFFCOMM\x12\0\0\0\0\x01', ValueError, 'truncated COMM'),
    (b'FORM\x04\0\0\08SVX', ValueError, 'not AIFF'),
    (pw.aiff(b'\0' * 8, 8000, 1, 4, 's16be')[:38], ValueError, 'no SSND chunk'),
    (pw.aiff(b'\0' * 8, 8000, 1, 4, 's16be', rate80=pw.ext80(11025.5)), NotImplementedError,
     'non-integer AIFF sample rate 11025.5'),
    (pw.aiff(b'\0' * 8, 8000, 1, 4, 's16be', rate80=b'\0' * 10), ValueError, 'not a positive finite'),
    (pw.aiff(b'\0' * 8, 8000, 1, 4, 's16be', comp=b'ima4'), NotImplementedError, "compression b'ima4'"),
    (pw.aiff(b'\0' * 8, 8000, 1, 2, 's32be', bits=48), NotImplementedError, '48-bit integer'),
    (pw.aiff(b'\0' * 18, 8000, 9, 1, 's16be'), NotImplementedError, '9 channels'),
])
def test_refusals_name_the_reason(data, exc, msg):
    from mvector.pcm import parse_header
    with pytest.raises(exc, match=msg):
        parse_header(data)


@pytest.mark.parametrize('data,exc,msg', [
    (_wav_fmt_only(2), NotImplementedError, 'Microsoft ADPCM'),
    (pw.wav(b'\0' * 30, 8000, 10, 's24le'), NotImplementedError, '10 channels'),
    (pw.wav(b'\0' * 8, 8000, 1, 'f32le'), None, None),
    (pw.aiff(b'\0' * 18, 8000, 9, 1, 's16be'), NotImplementedError, '9 channels'),
    (b'RIFF\x0c\0\0\0WAVEdata\0\0\0\0', ValueError, 'no fmt chunk'),
])
def test_segments_raise_the_parsers_error_when_wave_cannot_read_either(data, exc, msg):
    from mvector.audio import AudioSegment, PcmSegment
    if exc is None:
        assert isinstance(AudioSegment.from_bytes(data), PcmSegment)
        return
    with pytest.raises(exc, match=msg):
        AudioSegment.from_bytes(data)


def test_rows_past_2_31_samples_refused(tmp_path):
    """A 2^31-frame 8-bit WAV (a sparse file, mapped): refused from its header alone."""
    from mvector.pcm import parse_header
    n = 2 ** 31
    head = pw.wav(b'', 8000, 1, 'u8', data_size=n)
    p = tmp_path / 'big.wav'
    with open(p, 'wb') as f:
        f.write(head)
        f.truncate(len(head) + n)
    with open(p, 'rb') as f, mmap.mmap(f.fileno(), 0, access=mmap.ACCESS_READ) as m:
        with pytest.raises(NotImplementedError, match='2147483648 samples per channel'):
            parse_header(m)
        assert parse_header(m[:len(head) + 1000]).frames == 1000


def test_unknown_magic_still_goes_to_wave():
    from mvector.audio import AudioSegment
    with pytest.raises(wave.Error):
        AudioSegment.from_bytes(b'JUNK' + b'\0' * 60)


# ------------------------------------------------------------------------------------------------ no conversion
@pytest.fixture
def no_convert(monkeypatch):
    import mvector.audio as audio
    import mvector.pcm as pcm

    def boom(*a, **k):
        raise AssertionError('converted')
    monkeypatch.setattr(pcm, 'to_mono', boom)
    monkeypatch.setattr(audio.PcmSegment, 'decode_device', boom)


def test_segments_know_duration_without_converting(no_convert, tmp_path):
    from mvector.audio import AudioSegment, PcmSegment
    raw = pw.encode(pw.random_samples(np.random.default_rng(8), 's24le', 2 * 12345), 's24le')
    for name, data in (('a.wav', pw.wav(raw, 48000, 2, 's24le')), ('a.aif', pw.aiff(raw, 48000, 2, 12345, 's24le'))):
        p = tmp_path / name
        p.write_bytes(data)
        with open(p, 'rb') as f:
            segs = [AudioSegment.from_file(str(p)), AudioSegment.from_bytes(data), AudioSegment.from_file(f)]
        for s in segs:
            assert isinstance(s, PcmSegment)
            assert s.sample_rate == 48000 and s.duration == 12345 / 48000
        with pytest.raises(AssertionError, match='converted'):
            segs[0].samples


def test_eval_order_sorts_pcm_without_converting(no_convert, tmp_path):
    from mvector.trainer import MVectorTrainer
    rng = np.random.default_rng(9)
    lines, lens = [], []
    for i, n in enumerate((9000, 3000, 6000)):
        raw = pw.encode(pw.random_samples(rng, 'f32le', n), 'f32le')
        p = tmp_path / f'{i}.wav'
        p.write_bytes(pw.wav(raw, 16000, 1, 'f32le'))
        lines.append(f'{p}\t{i}\n')
    lst = tmp_path / 'list.txt'
    lst.write_text(''.join(lines))
    order = MVectorTrainer._eval_order(None, str(lst))
    assert [lab for _, lab in order] == [1, 2, 0]


def test_samples_setter_and_host_conditioning():
    from mvector.audio import AudioSegment
    vals = pw.random_samples(np.random.default_rng(10), 's16le', 8000)
    vals = (vals // 4).astype(np.int64)
    seg = AudioSegment.from_bytes(pw.wav(pw.encode(vals, 's16le'), 8000, 1, 's16le'))
    ref = AudioSegment(vals.astype(np.int16), 8000)
    seg.resample(16000)
    ref.resample(16000)
    seg.normalize(-20)
    ref.normalize(-20)
    assert seg.sample_rate == 16000 and np.array_equal(seg.samples, ref.samples)
    assert seg.duration == ref.duration == 1.0


# ------------------------------------------------------------------------------------------------ the wave path
def _wave_path(path):
    """The reader PcmSegment replaces for these files: wave + pcm_to_mono, 8-bit unsigned."""
    from mvector.audio import pcm_to_mono
    with wave.open(str(path), 'rb') as w:
        n, ch, sw = w.getnframes(), w.getnchannels(), w.getsampwidth()
        raw = w.readframes(n)
    ints = {1: lambda: np.frombuffer(raw, np.uint8).astype(np.int16) - 128, 2: lambda: np.frombuffer(raw, '<i2'),
            4: lambda: np.frombuffer(raw, '<i4')}[sw]()
    return pcm_to_mono(ints, ch, 8 * sw)


@pytest.mark.parametrize('sw', [1, 2, 4])
def test_stdlib_wave_files_bit_identical_to_the_wave_path(sw, tmp_path):
    from mvector.audio import AudioSegment, PcmSegment
    rng = np.random.default_rng(20 + sw)
    for ch in range(1, 9):
        n = int(rng.integers(100, 3000))
        vals = pw.random_samples(rng, {1: 'u8', 2: 's16le', 4: 's32le'}[sw], n * ch)
        p = tmp_path / f'{sw}_{ch}.wav'
        with wave.open(str(p), 'wb') as w:
            w.setnchannels(ch)
            w.setsampwidth(sw)
            w.setframerate(int(rng.choice([8000, 16000, 44100])))
            w.writeframes(pw.encode(vals, {1: 'u8', 2: 's16le', 4: 's32le'}[sw]))
        seg = AudioSegment.from_file(str(p))
        assert isinstance(seg, PcmSegment)
        ref = _wave_path(p)
        assert np.array_equal(_bits(seg.samples), _bits(ref)), (sw, ch)
        with wave.open(str(p), 'rb') as w:
            assert seg.sample_rate == w.getframerate() and seg.info.frames == w.getnframes()


@pytest.mark.parametrize('ch', [9, 12, 16])
def test_more_than_8_channel_int_wavs_keep_the_wave_path(ch, tmp_path):
    """Integer WAVs the PCM parser refuses for their channel count are read by the wave reader, as before it existed."""
    from mvector.audio import AudioSegment, PcmSegment
    rng = np.random.default_rng(60 + ch)
    for sw, fmt in ((1, 'u8'), (2, 's16le'), (4, 's32le')):
        p = tmp_path / f'{ch}_{sw}.wav'
        with wave.open(str(p), 'wb') as w:
            w.setnchannels(ch)
            w.setsampwidth(sw)
            w.setframerate(16000)
            w.writeframes(pw.encode(pw.random_samples(rng, fmt, 100 * ch), fmt))
        ref = _wave_path(p)
        with open(p, 'rb') as f:
            segs = [AudioSegment.from_file(str(p)), AudioSegment.from_bytes(p.read_bytes()), AudioSegment.from_file(f)]
        for seg in segs:
            assert not isinstance(seg, PcmSegment) and seg.sample_rate == 16000
            assert np.array_equal(_bits(seg.samples), _bits(ref)), (ch, sw)


def test_contradicting_block_align_keeps_the_wave_path(tmp_path):
    """A 16-bit WAV whose block align contradicts its channels: the parser refuses it, the wave reader (which ignores
    block align) reads it as before."""
    from mvector.audio import AudioSegment, PcmSegment
    vals = pw.random_samples(np.random.default_rng(61), 's16le', 2 * 300)
    data = pw.wav(pw.encode(vals, 's16le'), 16000, 2, 's16le', block_align=6)
    p = tmp_path / 'align.wav'
    p.write_bytes(data)
    seg = AudioSegment.from_bytes(data)
    assert not isinstance(seg, PcmSegment)
    assert np.array_equal(_bits(seg.samples), _bits(_wave_path(p)))
