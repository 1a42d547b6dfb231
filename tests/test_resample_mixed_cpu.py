"""CPU: the mixed streams call (fs2_resample_streams_mixed): its ABI and refusals (every refusal happens before any CUDA call), a numpy
ITU-T G.711 oracle checked against audioop, and StreamPool's bookkeeping with streams of different rates and encodings through a
substituted launch and conversion call."""
import ctypes
import warnings

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L
from fastspeech2_b200.hifigan.models import StreamPool
from fastspeech2_b200.resample import ENCODINGS, Resampler

FS_IN = 22050

# G.711 segment end points (the largest magnitude of each of the eight segments)
_ULAW_END = np.array([0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF, 0x1FFF])
_ALAW_END = np.array([0x1F, 0x3F, 0x7F, 0xFF, 0x1FF, 0x3FF, 0x7FF, 0xFFF])


def ulaw_ref(pcm):
    """mu-law bytes of int16 samples (ITU-T G.711): the 14-bit sample s >> 2, magnitude clipped to 8159 and biased by 33, its segment
    and four mantissa bits below the segment's leading bit, all bits inverted, sign bit set for non-negative samples."""
    v = np.asarray(pcm, dtype=np.int64) >> 2
    mag = np.minimum(np.abs(v), 8159) + 33
    seg = np.searchsorted(_ULAW_END, mag)                     # first segment whose end is >= mag; 8 past the last
    code = np.where(seg >= 8, 0x7F, (np.minimum(seg, 7) << 4) | ((mag >> (np.minimum(seg, 7) + 1)) & 0xF))
    return (code ^ np.where(v < 0, 0x7F, 0xFF)).astype(np.uint8)


def alaw_ref(pcm):
    """A-law bytes of int16 samples (ITU-T G.711): the 13-bit sample s >> 3, magnitude -v - 1 for negative v, its segment and four
    mantissa bits (bits 1..4 in the first two segments), even bits inverted, sign bit set for non-negative samples."""
    v = np.asarray(pcm, dtype=np.int64) >> 3
    mag = np.where(v < 0, -v - 1, v)
    seg = np.searchsorted(_ALAW_END, mag)
    code = (seg << 4) | ((mag >> np.where(seg < 2, 1, seg)) & 0xF)
    return (code ^ np.where(v < 0, 0x55, 0xD5)).astype(np.uint8)


def g711_ref(pcm, encoding):
    return {L.RESAMPLE_ULAW: ulaw_ref, L.RESAMPLE_ALAW: alaw_ref}[encoding](pcm)


ALL_INT16 = np.arange(-32768, 32768, dtype=np.int64)


def test_abi_of_the_mixed_call():
    h = L.lib()
    assert h.fs2_abi_version() == L.ABI_VERSION == 12
    assert hasattr(h, "fs2_resample_streams_mixed")
    assert ctypes.sizeof(L.ResampleFilter) == L.RESAMPLE_FILTER_SIZE == 24
    assert ctypes.sizeof(L.ResampleMixedStream) == L.RESAMPLE_MIXED_STREAM_SIZE == 80
    assert ctypes.sizeof(L.ResampleMixedArgs) == L.RESAMPLE_MIXED_ARGS_SIZE == 232
    assert [f[0] for f in L.ResampleMixedStream._fields_] == ["x0", "x1", "i0", "i1", "i2", "n", "j0", "j1", "filter", "encoding",
                                                             "y_offset"]
    assert L.ResampleMixedArgs.filters.offset == 8 and L.ResampleMixedArgs.table.offset == 200
    assert (L.RESAMPLE_MAX_FILTERS, L.RESAMPLE_F32, L.RESAMPLE_PCM16, L.RESAMPLE_ULAW, L.RESAMPLE_ALAW) == (8, 0, 1, 2, 3)
    assert [h.fs2_struct_size(i) > 0 for i in range(19)] == [True] * 19 and h.fs2_struct_size(19) == 0


def _mixed(n_filters=2, filters=None, **kw):
    """Args of a call that the host accepts (a 16 kHz filter and the identity) but for the fields in kw."""
    a16 = Resampler(FS_IN, 16000)
    good = [dict(up=a16.up, down=a16.down, K=a16.K, taps=0x1000), dict(up=1, down=1, K=1, taps=0x2000)]
    a = L.ResampleMixedArgs(B=3, n_filters=n_filters, table=0x1000, max_out=64, y=0x1000, scale=32768.0)
    for i, f in enumerate(filters or good):
        a.filters[i] = L.ResampleFilter(**f)
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def test_mixed_refusals():
    h = L.lib()
    call = lambda a: h.fs2_resample_streams_mixed(ctypes.byref(a), None)
    rs = Resampler(FS_IN, 16000)
    f16 = dict(up=rs.up, down=rs.down, K=rs.K, taps=0x1000)
    for kw in (dict(B=0), dict(B=65536), dict(n_filters=0), dict(n_filters=9), dict(table=0), dict(max_out=0), dict(max_out=-1),
               dict(y=0), dict(y=0x1008), dict(y=0x1001)):
        assert call(_mixed(**kw)) == -1, kw
    bad_filters = (
        dict(f16, K=rs.K + 1), dict(f16, taps=0), dict(f16, up=0), dict(f16, down=-1), dict(f16, up=640, down=882),
        dict(f16, up=2049), dict(up=1, down=1, K=21, taps=0x1000), dict(up=1, down=1, K=0, taps=0x1000),
        dict(up=1, down=1, K=1, taps=0),
    )
    for f in bad_filters:
        assert call(_mixed(filters=[f16, f])) == -1, f
        assert call(_mixed(n_filters=1, filters=[f])) == -1, f
    a = L.ResampleStreamsArgs(B=1, up=1, down=1, K=1, taps=0x1000, table=0x1000, max_out=8, y=0x1000, y_batch_stride=8, pcm16=1,
                              scale=1.0)
    assert h.fs2_resample_streams(ctypes.byref(a), None) == -1            # the identity stays refused by the older calls


def test_g711_oracle_against_audioop():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        try:
            import audioop
        except ImportError:
            pytest.skip("audioop is not available in this Python")
    raw = ALL_INT16.astype("<i2").tobytes()
    assert np.array_equal(ulaw_ref(ALL_INT16), np.frombuffer(audioop.lin2ulaw(raw, 2), dtype=np.uint8))
    assert np.array_equal(alaw_ref(ALL_INT16), np.frombuffer(audioop.lin2alaw(raw, 2), dtype=np.uint8))


def test_g711_oracle_known_codes():
    """Codes of the standard's tables: zero, and positive and negative full scale; every code is reached except mu-law's negative
    zero 0x7F, which no encoder emits."""
    assert list(ulaw_ref([0, 32767, -32768])) == [0xFF, 0x80, 0x00]
    assert list(alaw_ref([0, 32767, -32768])) == [0xD5, 0xAA, 0x2A]
    assert set(range(256)) - set(ulaw_ref(ALL_INT16).tolist()) == {0x7F}
    assert len(np.unique(alaw_ref(ALL_INT16))) == 256


def test_mixed_table():
    """Filters in order of first use, shared by ratio; offsets back to back, 16-byte aligned, sized by each encoding; widths clamped
    to max_out."""
    r16, r8, r22 = Resampler(FS_IN, 16000), Resampler(FS_IN, 8000), Resampler(FS_IN, FS_IN)
    r16b = Resampler(FS_IN, 16000)
    recs = [(1, 2, 0, 0, 10, 100, 0, 7, r16, L.RESAMPLE_F32),
            (3, 4, 0, 0, 10, 100, 5, 18, r8, L.RESAMPLE_ULAW),
            (5, 6, 0, 0, 10, 100, 0, 9, r22, L.RESAMPLE_PCM16),
            (7, 8, 0, 0, 10, 100, 0, 0, r16b, L.RESAMPLE_ALAW),
            (9, 10, 0, 0, 10, 100, 3, 40, r16, L.RESAMPLE_PCM16)]
    filters, table, offsets, nbytes = Resampler.mixed_table(recs, max_out=20)
    assert filters == [r16, r8, r22]
    assert offsets == [0, 32, 48, 80, 80] and nbytes == 128
    assert table[:, 8].tolist() == [0, 1 | 2 << 32, 2 | 1 << 32, 0 | 3 << 32, 0 | 1 << 32]
    assert table[:, 9].tolist() == offsets and table[:, :8].tolist() == [list(r[:8]) for r in recs]
    with pytest.raises(ValueError):
        Resampler.mixed_table([recs[0][:9] + (7,)], 20)
    many = [(0, 0, 0, 0, 1, 1, 0, 1, Resampler(FS_IN, r), L.RESAMPLE_F32) for r in (8000, 11025, 12000, 16000, 24000, 32000, 44100,
                                                                                    48000, 96000)]
    Resampler.mixed_table(many[:8], 1)
    with pytest.raises(ValueError):
        Resampler.mixed_table(many, 1)


class FakeConvert:
    """Records each step's records and returns rows that name (stream, output index) so the chunks can be checked."""

    def __init__(self, rs):
        self.rs, self.calls = rs, []

    def __call__(self, records, max_out):
        self.calls.append(records)
        return [torch.arange(r[6], r[6] + max_out, dtype=torch.float64) + 1e6 * r[5] for r in records]


def _mixed_pool(chunk=2, up=256, default=FS_IN, encoding="f32"):
    convert = FakeConvert(Resampler(FS_IN, default))
    launches = []

    def launch(ptrs, f0s, ns):
        launches.append(list(ns))
        return torch.zeros(len(ptrs), chunk * up)
    return StreamPool(launch, 80, up, chunk, "cpu", resample=convert, encoding=encoding), convert, launches


FORMATS = ((8000, "ulaw"), (8000, "alaw"), (16000, "pcm16"), (22050, "pcm16"), (22050, "f32"), (24000, "f32"), (44100, "pcm16"),
           (48000, "f32"))


def test_pool_bookkeeping_with_mixed_formats():
    up, chunk = 256, 2
    pool, convert, launches = _mixed_pool(chunk, up)
    lens = (5, 1, 3, 4, 6, 2, 7, 3)
    hs = [pool.add(torch.zeros(80, n), sample_rate=r, encoding=e) for n, (r, e) in zip(lens, FORMATS)]
    got = {h: [] for h in hs}
    n_steps = 0
    while len(pool):
        for h, start, y in pool.step():
            got[h].append((start, y.shape[2]))
            assert y.shape[:2] == (1, 1)
        n_steps += 1
    assert len(convert.calls) == n_steps == max(-(-n // chunk) for n in lens)
    for h, n, (rate, enc) in zip(hs, lens, FORMATS):
        rs = Resampler(FS_IN, rate)
        starts = [s for s, _ in got[h]]
        assert len(got[h]) == -(-n // chunk)
        assert starts[0] == 0 and all(s + w == s2 for (s, w), s2 in zip(got[h], starts[1:]))
        assert sum(w for _, w in got[h]) == rs.n_out(n * up)
    first = convert.calls[0]
    # stream 4 (22 050 Hz fp32) takes its slice of the waveform and is absent from the conversion call
    assert len(first) == 7
    assert [(r[8].fs_out, r[9]) for r in first] == [(r, ENCODINGS[e]) for r, e in FORMATS if (r, e) != (FS_IN, "f32")]
    assert all(r[2:6] == (0, 0, chunk * up, n * up) and r[0] == 0 for r, n in zip(first, lens[:4] + lens[5:]))
    second = convert.calls[1]
    assert second[0][0] == first[0][1] and second[0][2:5] == (0, chunk * up, 2 * chunk * up) and second[0][6] == first[0][7]
    # the table the conversion call builds from these records: eight streams' seven rates -> six filters, the identity among them
    filters, table, _, _ = Resampler.mixed_table(first, max(r[7] - r[6] for r in first))
    assert [f.fs_out for f in filters] == [8000, 16000, 22050, 24000, 44100, 48000]
    assert (table[:, 8] & 0xFFFFFFFF).tolist() == [0, 0, 1, 2, 3, 4, 5] and (table[:, 8] >> 32).tolist() == [2, 3, 1, 1, 0, 1, 0]


def test_pool_without_conversions_makes_no_call():
    pool, convert, launches = _mixed_pool()
    pool.add(torch.zeros(80, 3))
    pool.add(torch.zeros(80, 2), sample_rate=FS_IN, encoding="f32")
    while len(pool):
        for _, _, y in pool.step():
            assert y.dtype == torch.float32
    assert convert.calls == [] and len(launches) == 2
    pool, convert, _ = _mixed_pool(default=16000, encoding="pcm16")   # the pool's defaults convert; a native fp32 stream does not
    pool.add(torch.zeros(80, 3), sample_rate=FS_IN, encoding="f32")
    pool.add(torch.zeros(80, 3))
    pool.step()
    assert len(convert.calls) == 1 and [(r[8].fs_out, r[9]) for r in convert.calls[0]] == [(16000, L.RESAMPLE_PCM16)]


def test_pool_add_refusals():
    pool, _, _ = _mixed_pool(chunk=123)
    for rate in (0, -8000, 8000.5, True, "8000", 1):          # 22 050 -> 1 Hz: max(up, down) > 2048
        with pytest.raises(ValueError):
            pool.add(torch.zeros(80, 3), sample_rate=rate)
    with pytest.raises(ValueError):
        pool.add(torch.zeros(80, 3), sample_rate=14)           # K - 1 = 31500 > 123 * 256
    for enc in ("mp3", "PCM16", 1, "u-law"):
        with pytest.raises(ValueError):
            pool.add(torch.zeros(80, 3), encoding=enc)
    pool, _, _ = _mixed_pool()
    rates = (8000, 11025, 12000, 16000, 24000, 32000, 44100, 48000)
    hs = [pool.add(torch.zeros(80, 3), sample_rate=r) for r in rates]
    pool.add(torch.zeros(80, 3), sample_rate=8000, encoding="alaw")      # a live rate: accepted
    with pytest.raises(ValueError):
        pool.add(torch.zeros(80, 3), sample_rate=96000)                   # a ninth
    with pytest.raises(ValueError):
        pool.add(torch.zeros(80, 3))                                      # the default, 22 050 Hz, is a ninth too
    pool.cancel(hs[0])
    with pytest.raises(ValueError):
        pool.add(torch.zeros(80, 3), sample_rate=96000)                   # 8 000 Hz is still live: the A-law stream
    pool.cancel(hs[1])
    pool.add(torch.zeros(80, 3), sample_rate=96000)                       # 11 025 Hz has left
    with pytest.raises(ValueError):
        pool.add(torch.zeros(80, 3), sample_rate=22050)
    assert len(pool) == 8
    plain = StreamPool(lambda p, f, n: torch.zeros(len(p), 8), 80, 4, 2, "cpu")
    for kw in (dict(sample_rate=16000), dict(encoding="pcm16"), dict(encoding="ulaw")):
        with pytest.raises(ValueError):
            plain.add(torch.zeros(80, 3), **kw)
    plain.add(torch.zeros(80, 3), encoding="f32")
    with pytest.raises(ValueError):
        StreamPool(lambda p, f, n: None, 80, 4, 2, "cpu", encoding="pcm16")
