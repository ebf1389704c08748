"""FLAC on the host: the CRCs, known-answer frames assembled bit by bit from RFC 9639's field tables, the test encoder
against the Python decoder over the feature matrix, the STREAMINFO parser, and segments that know their length
without decoding."""
import io

import numpy as np
import pytest

import flac_cases
import flac_oracle as fo
import flac_writer as fw


def test_crc_check_values():
    assert fw.crc8(b'123456789') == 0xF4
    assert fw.crc16(b'123456789') == 0xFEE8


def _stream(frames_bits, rate=16000, ch=1, bps=16, total=None, min_bs=16, max_bs=4096):
    """STREAMINFO + frames given as bit strings (header through subframes, before padding and CRC-16)."""
    out = b'fLaC' + bytes([0x80, 0, 0, 34]) + fw._streaminfo(min_bs, max_bs, 0, 0, rate, ch, bps, total)
    for bits in frames_bits:
        bits = bits.replace(' ', '')
        bits += '0' * (-len(bits) % 8)
        body = int(bits, 2).to_bytes(len(bits) // 8, 'big')
        out += body + fw.crc16(body).to_bytes(2, 'big')
    return out


def _hdr(b2, b3, num_bytes, extra=b''):
    h = bytes([0xFF, 0xF8 if num_bytes[0] != 'v' else 0xF9, b2, b3]) + bytes(num_bytes[1]) + extra
    h += bytes([fw.crc8(h)])
    return ''.join(f'{x:08b}' for x in h)


def test_known_answer_constant_and_verbatim():
    # frame 0: block size code 6 (8-bit escape, 4 samples), rate code 5 (16 kHz), mono, 16 bit; CONSTANT -3
    f0 = _hdr(0x65, 0x08, ('f', [0]), bytes([3])) + '0 000000 0' + f'{(-3) & 0xFFFF:016b}'
    # frame 1: VERBATIM 1, -2, 32767, -32768
    f1 = _hdr(0x65, 0x08, ('f', [1]), bytes([3])) + '0 000001 0' + ''.join(
        f'{v & 0xFFFF:016b}' for v in (1, -2, 32767, -32768))
    data = _stream([f0, f1], total=8, min_bs=16, max_bs=4)
    ints, _ = fo.decode(data)
    assert ints[:, 0].tolist() == [-3, -3, -3, -3, 1, -2, 32767, -32768]


def test_known_answer_fixed2_rice_and_escape():
    # 8 samples, 16-bit escape of the block size, FIXED order 2, warm-up 10, 20; residual method 0, partition order 1:
    # partition 0 (4 - 2 = 2 residuals) Rice k=1: 0 -> u=0 '1'+'0', -1 -> u=1 '1'+'1'; partition 1 escaped, 3 bits: 1, -2, 3, 0
    hdr = _hdr(0x75, 0x08, ('f', [0]), bytes([0, 7]))
    sub = '0 001010 0' + f'{10:016b}' + f'{20:016b}' + '00' + '0001' + '0001' + '10' + '11' + '1111' + '00011' + \
        '001' + '110' + '011' + '000'
    data = _stream([hdr + sub], total=8, min_bs=16, max_bs=8)
    ints, _ = fo.decode(data)
    # predictions 2 x[i-1] - x[i-2]: 30 (+0), 40 (-1 -> 39), 2*39-30=48 (+1), 2*49-39=59 (-2 -> 57), 65 (+3 -> 68), 79 (+0)
    assert ints[:, 0].tolist() == [10, 20, 30, 39, 49, 57, 68, 79]


def test_known_answer_lpc1_mid_side_wasted_rate_escape_variable():
    # variable blocking, sample number 200 (2 bytes: 0xC3 0x88), block size code 6 (2 samples), rate code 12 (8 kHz)
    # stereo mid/side (assign 10), 8 bit; mid: LPC order 1, precision 2, shift 1, coef 1 -> pred x[i-1] >> 1;
    # side: VERBATIM with 1 wasted bit (9 - 1 = 8 bits per sample)
    hdr = _hdr(0x6C, 0xA2, ('v', [0xC3, 0x88]), bytes([1, 8]))
    mid = '0 100000 0' + f'{20:08b}' + '0001' + '00001' + '01' + '00' + '0000' + '0001' + '11'  # resid -1 -> u=1, k=1
    side = '0 000001 1 1' + f'{(-4 >> 1) & 0xFF:08b}' + f'{(6 >> 1) & 0xFF:08b}'
    first = _hdr(0x6C, 0xA2, ('v', [0]), bytes([199, 8])) + '0 000000 0' + f'{0:08b}' + '0 000000 0' + f'{0:09b}'
    data = _stream([first, hdr + mid + side], rate=8000, ch=2, bps=8, total=202, min_bs=16, max_bs=200)
    ints, _ = fo.decode(data)
    # mid 20, (20 >> 1) - 1 = 9; side -4, 6: m = (mid << 1) | (side & 1) -> 40, 18; L = (m + s) >> 1, R = (m - s) >> 1
    assert ints[200:].tolist() == [[18, 22], [12, 6]]


def test_encoder_round_trip_matrix():
    for name, data, pcm, bps in flac_cases.matrix(seed=1):
        ints, info = fo.decode(data)
        assert np.array_equal(ints, pcm), name


def test_fake_sync_in_payload():
    rng = np.random.default_rng(4)
    pcm = flac_cases.fake_sync_pcm(rng)
    data = fw.encode(pcm, 16000, 8, blocksize=256, sub=lambda fi, c, x: dict(kind='verbatim'))
    fake = flac_cases.fake_headers(dict(rate=16000, bps=8))
    assert data.count(fake) >= 4
    assert np.array_equal(fo.decode(data)[0], pcm)


def test_pcm_to_mono_matches_numpy_mean_for_1_to_8_channels():
    from mvector.audio import pcm_to_mono
    rng = np.random.default_rng(0)
    for ch in range(1, 9):
        ints = rng.integers(-2 ** 23, 2 ** 23, size=(5000, ch))
        got = pcm_to_mono(ints.reshape(-1), ch, 24)
        x = ints.astype(np.float32) / np.float32(2 ** 23)
        if ch < 8:
            s = x[:, 0].copy()
            for c in range(1, ch):
                s = s + x[:, c]
        else:
            s = ((x[:, 0] + x[:, 1]) + (x[:, 2] + x[:, 3])) + ((x[:, 4] + x[:, 5]) + (x[:, 6] + x[:, 7]))
        assert np.array_equal(got.view(np.int32), (s / np.float32(ch)).view(np.int32)), ch


# ------------------------------------------------------------------------------------------------ metadata
def test_streaminfo_fields_and_skipped_blocks():
    from mvector.flac import parse_streaminfo
    pcm = fw.random_pcm(np.random.default_rng(0), 5000, 2, 20)
    data = fw.encode(pcm, 44100, 20, blocksize=1152, extra_blocks=[(4, b'\0' * 40), (1, b'\0' * 7)])
    si = parse_streaminfo(data)
    assert (si.sample_rate, si.channels, si.bps, si.total_samples) == (44100, 2, 20, 5000)
    assert (si.min_blocksize, si.max_blocksize) == (1152, 1152)
    assert si.frame_offset == 4 + 4 + 34 + 4 + 40 + 4 + 7
    assert data[si.frame_offset] == 0xFF
    assert si.max_framesize > 0 and si.duration == 5000 / 44100


def test_streaminfo_refusals():
    from mvector.flac import parse_streaminfo
    good = fw.encode(fw.random_pcm(np.random.default_rng(0), 500, 1, 16), 16000, 16, blocksize=256)
    with pytest.raises(ValueError, match='truncated'):
        parse_streaminfo(good[:20])
    with pytest.raises(ValueError, match='magic'):
        parse_streaminfo(b'RIFF' + good[4:])
    with pytest.raises(NotImplementedError, match='Ogg'):
        parse_streaminfo(b'OggS' + good[4:])
    with pytest.raises(NotImplementedError, match='ID3'):
        parse_streaminfo(b'ID3\x04' + good)
    zero = bytearray(good)
    v = int.from_bytes(zero[18:26], 'big') & ~((1 << 36) - 1)
    zero[18:26] = v.to_bytes(8, 'big')
    with pytest.raises(NotImplementedError, match='unknown length'):
        parse_streaminfo(bytes(zero))
    b32 = bytearray(good)
    v = (int.from_bytes(b32[18:26], 'big') & ~(31 << 36)) | (31 << 36)
    b32[18:26] = v.to_bytes(8, 'big')
    with pytest.raises(NotImplementedError, match='32-bit'):
        parse_streaminfo(bytes(b32))
    with pytest.raises(ValueError, match='STREAMINFO'):
        parse_streaminfo(b'fLaC' + bytes([0x84, 0, 0, 2, 0, 0]) + good[42:])


@pytest.fixture
def no_decode(monkeypatch):
    import mvector.audio as audio

    def boom(*a, **k):
        raise AssertionError('decoded')
    monkeypatch.setattr(audio, 'decode_segments', boom)
    monkeypatch.setattr(audio.FlacSegment, 'decode_device', boom)


def test_segments_know_duration_without_decoding(no_decode, tmp_path):
    from mvector.audio import AudioSegment, FlacSegment
    pcm = fw.random_pcm(np.random.default_rng(1), 12345, 2, 16)
    data = fw.encode(pcm, 48000, 16, blocksize=4096)
    p = tmp_path / 'a.flac'
    p.write_bytes(data)
    with open(p, 'rb') as f:
        segs = [AudioSegment.from_file(str(p)), AudioSegment.from_bytes(data), AudioSegment.from_file(f)]
    for s in segs:
        assert isinstance(s, FlacSegment)
        assert s.sample_rate == 48000 and s.duration == 12345 / 48000
    with pytest.raises(AssertionError, match='decoded'):
        segs[0].samples


def test_eval_order_sorts_flac_without_decoding(no_decode, tmp_path):
    from mvector.trainer import MVectorTrainer
    rng = np.random.default_rng(2)
    lines = []
    for i, n in enumerate([9000, 3000, 6000, 1000]):
        p = tmp_path / f'{i}.flac'
        p.write_bytes(fw.encode(fw.random_pcm(rng, n, 1, 16), 16000, 16, blocksize=4096))
        lines.append(f'{p}\t{i}\n')
    lst = tmp_path / 'list.txt'
    lst.write_text(''.join(lines))
    order = MVectorTrainer._eval_order(None, str(lst))
    assert [lb for _, lb in order] == [3, 1, 2, 0]


def test_wav_decoding_unchanged(tmp_path):
    import wave
    from mvector.audio import AudioSegment
    rng = np.random.default_rng(3)
    for sw, ch in ((1, 1), (2, 2), (4, 3), (2, 8)):
        dt = {1: np.uint8, 2: '<i2', 4: '<i4'}[sw]
        info = np.iinfo(np.dtype(dt))
        raw = rng.integers(info.min, info.max, size=(777, ch), endpoint=True).astype(dt)
        p = tmp_path / f'{sw}-{ch}.wav'
        with wave.open(str(p), 'wb') as w:
            w.setnchannels(ch); w.setsampwidth(sw); w.setframerate(16000); w.writeframes(raw.tobytes())
        if sw == 1:
            ref = (raw.astype(np.float32) - 128.0) / 128.0
        else:
            ref = raw.astype(np.float32) / float(2 ** (8 * sw - 1))
        if ch > 1:
            ref = ref.reshape(-1, ch).mean(axis=1)
        for seg in (AudioSegment.from_file(str(p)), AudioSegment.from_bytes(p.read_bytes()),
                    AudioSegment.from_file(io.BytesIO(p.read_bytes()))):
            assert np.array_equal(seg.samples.view(np.int32), ref.reshape(-1).view(np.int32))
