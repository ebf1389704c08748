"""Host halves of the device diarization front (csrc/segment.cu, MVectorPredictor.speaker_diarization): the summation
order vp_frame_energy restates against numpy's own frame energies, the VAD split into energies and decision, and
SpeakerDiarization.chunk_table against the slicing segmentation it replaces, including every assert."""
import numpy as np
import pytest


def pairwise_sum(a):
    """numpy's pairwise sum of a float64 sequence (the order vp_frame_energy reproduces)."""
    n = len(a)
    if n < 8:
        r = 0.0
        for v in a:
            r += v
        return r
    if n <= 128:
        r = [float(v) for v in a[:8]]
        m = n - n % 8
        for i in range(8, m, 8):
            for j in range(8):
                r[j] += a[i + j]
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for i in range(m, n):
            res += a[i]
        return res
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(a[:n2]) + pairwise_sum(a[n2:])


# below 8, 8 .. 128, and above 128 -- 129, 441 and 1323 split unevenly (n2 = n/2 - (n/2) % 8 != n - n2)
@pytest.mark.parametrize('hop', [1, 3, 7, 8, 9, 64, 100, 127, 128, 129, 200, 441, 480, 1323, 1440, 2000])
def test_pairwise_restatement_equals_numpy_frame_energy(hop):
    rng = np.random.default_rng(hop)
    x = (rng.standard_normal(hop * 5 + hop // 2) * rng.uniform(1e-4, 3)).astype(np.float32)
    nf = x.size // hop
    X = x[:nf * hop].astype(np.float64).reshape(nf, hop)
    ref = (X ** 2).mean(axis=1)
    mine = np.array([pairwise_sum(list(r * r)) / hop for r in X])
    assert np.array_equal(ref.view(np.uint64), mine.view(np.uint64))


def test_vad_equals_vad_from_host_energies():
    from mvector.audio import AudioSegment
    rng = np.random.RandomState(1)
    for sr in (8000, 16000, 44100, 48000):
        parts = []
        for _ in range(12):
            parts.append(np.zeros(int(sr * rng.uniform(0.05, 0.8)), dtype=np.float32))
            parts.append((rng.uniform(0.001, 0.3) * rng.randn(int(sr * rng.uniform(0.1, 2.0)))).astype(np.float32))
        seg = AudioSegment(np.concatenate(parts), sr)
        ms = seg.frame_energy()
        n = seg.samples.shape[0]
        assert ms.shape == (n // AudioSegment.vad_hop(sr),)
        for secs in (False, True):
            assert seg.vad(return_seconds=secs) == AudioSegment.vad_from_energy(ms, n, sr, return_seconds=secs)
    short = AudioSegment(np.ones(100, dtype=np.float32), 16000)
    assert short.vad() == [] == AudioSegment.vad_from_energy(short.frame_energy(), 100, 16000)


# ------------------------------------------------------------------------------------------------ chunk table
def _slicing_segments(vad_times, samples, sr, seg_duration=1.5, seg_shift=0.75):
    """The slicing segmentation chunk_table replaces: VAD slices of the samples, their checks, then the 1.5 s cut."""
    voiced = []
    for t in vad_times:
        st, ed = round(t['start'], 3), round(t['end'], 3)
        voiced.append([st, ed, samples[int(st * sr):int(ed * sr)]])
    total = 0
    for i, (st, ed, data) in enumerate(voiced):
        assert ed >= st, '分割的时间戳错误'
        assert isinstance(data, np.ndarray), '数据的类型不正确'
        assert int(ed * sr) - int(st * sr) == data.shape[0], '时间长度和数据长度不匹配'
        if i > 0:
            assert st >= voiced[i - 1][1], 'modelscope error: Wrong time stamps.'
        total += ed - st
    assert total > 5, f'音频时间过段，应当大于5秒，当前长度是{total}秒'
    size, hop = int(seg_duration * sr), int(seg_shift * sr)
    out = []
    for seg_st, _, data in voiced:
        n = data.shape[0]
        prev_end = 0
        for lo in range(0, n, hop):
            hi = min(lo + size, n)
            if hi <= prev_end:
                break
            prev_end = hi
            lo = max(0, hi - size)
            piece = data[lo:hi]
            if piece.shape[0] < size:
                piece = np.pad(piece, (0, size - piece.shape[0]), 'constant')
            out.append([lo / sr + seg_st, hi / sr + seg_st, piece])
    return out


def _outcome(fn):
    try:
        return 'ok', fn()
    except AssertionError as e:
        return 'assert', str(e).splitlines()[0]          # pytest appends its own explanation to asserts in this file


def _check_same(vad_times, samples, sr):
    from mvector.infer_utils.speaker_diarization import SpeakerDiarization
    from mvector.audio import AudioSegment
    kind, ref = _outcome(lambda: _slicing_segments(vad_times, samples, sr))
    sd = SpeakerDiarization()
    kt, table = _outcome(lambda: sd.chunk_table(vad_times, samples.shape[0], sr))
    assert kt == kind
    if kind == 'assert':
        assert table == ref
        return kind
    assert table.size == int(1.5 * sr) and len(table.start) == len(ref)
    for i, (st, ed, piece) in enumerate(ref):
        assert table.start[i] == st and table.end[i] == ed            # same float64 bits
        row = np.zeros(table.size, dtype=np.float32)                  # vp_gather_windows' row
        v = int(table.valid[i])
        row[:v] = samples[table.offset[i]:table.offset[i] + v]
        assert np.array_equal(row, piece) and piece.dtype == row.dtype
    # segments_audio on the same VAD: the same list
    seg = AudioSegment(samples, sr)
    seg.vad = lambda return_seconds=False: vad_times
    got = SpeakerDiarization().segments_audio(seg)
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        assert g[0] == r[0] and g[1] == r[1] and np.array_equal(g[2], r[2])
    return kind


def test_chunk_table_reproduces_slicing_on_random_vad_layouts():
    rng = np.random.RandomState(7)
    kinds = []
    for trial in range(300):
        sr = int(rng.choice([8000, 16000, 22050, 44100, 48000]))
        n = int(sr * rng.uniform(4.0, 40.0))
        samples = rng.randn(n).astype(np.float32)
        hop = max(1, int(sr * 0.03))
        t, times = 0, []
        while True:                              # VAD-like segments: frame multiples, the last one clipped to n
            a = t + int(rng.randint(0, 40)) * hop
            b = a + int(rng.randint(1, 200)) * hop
            if a >= n:
                break
            times.append({'start': a / sr, 'end': min(b, n) / sr})
            t = b
        kinds.append(_check_same(times, samples, sr))
    assert kinds.count('ok') > 100 and kinds.count('assert') > 10


def test_chunk_table_edges():
    sr = 16000
    x = np.random.RandomState(3).randn(sr * 30).astype(np.float32)

    def sec(a, b):
        return {'start': a, 'end': b}
    # a segment shorter than one chunk (zero padded), segments whose length is no multiple of the hop (the last chunk
    # right-aligned), a 1.5 s segment exactly, and a segment ending at the recording's end
    assert _check_same([sec(0.2, 1.0), sec(1.5, 5.123), sec(6.0, 7.5), sec(8.0, 30.0)], x, sr) == 'ok'
    # an empty segment contributes no chunk
    assert _check_same([sec(0.5, 0.5), sec(1.0, 9.0)], x, sr) == 'ok'
    # rounding to milliseconds moves int(ed sr) past the end: the slice is shorter than the times say
    n = 16000 * 7 + 9
    assert _check_same([sec(0.0, n / sr)], x[:n], sr) == 'assert'
    # < 5 s of speech, reversed times, overlapping segments
    for times in ([sec(0.0, 2.0), sec(3.0, 5.5)], [sec(0.0, 6.0), sec(7.0, 6.5)], [sec(0.0, 6.0), sec(5.0, 9.0)]):
        assert _check_same(times, x, sr) == 'assert'
    # offsets keep their int64 width
    from mvector.infer_utils.speaker_diarization import SpeakerDiarization
    t = SpeakerDiarization().chunk_table([sec(0.0, 10.0)], 160000, sr)
    assert t.offset.dtype == np.int64 and t.valid.dtype == np.int32
    assert t.offset.tolist()[-1] + int(t.valid[-1]) == 160000
