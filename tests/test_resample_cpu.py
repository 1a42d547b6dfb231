"""CPU: the resampler's tap design and oracle against scipy.signal, the streaming emission rule, argument checks, and the C ABI's
structs and refusals (every refusal happens before any CUDA call, so no GPU is needed)."""
import ctypes

import numpy as np
import pytest
import scipy.signal
import torch

from fastspeech2_b200 import _lib as L
from fastspeech2_b200.hifigan.models import StreamPool
from fastspeech2_b200.resample import Resampler, design_taps
from oracle.resample_ref import resample_ref

FS_IN = 22050
RATES = {16000: (320, 441), 48000: (320, 147), 24000: (160, 147), 44100: (2, 1), 8000: (160, 441)}


@pytest.mark.parametrize("fs_out", list(RATES))
def test_ratio_and_taps_match_scipy(fs_out):
    rs = Resampler(FS_IN, fs_out)
    assert (rs.up, rs.down) == RATES[fs_out]
    mx = max(rs.up, rs.down)
    want = scipy.signal.firwin(2 * 10 * mx + 1, 1.0 / mx, window=("kaiser", 5.0)) * rs.up
    got = design_taps(rs.up, rs.down)
    assert np.abs(got - want).max() <= 1e-15 * rs.up
    assert rs.K == -(-len(want) // rs.up) and rs.taps.shape == (rs.up, rs.K) and rs.taps.dtype == np.float32
    for p in (0, rs.up // 2, rs.up - 1):                       # polyphase rows, zero-filled past the filter
        row = want[p::rs.up].astype(np.float32)
        assert np.array_equal(rs.taps[p, :len(row)], row) and not rs.taps[p, len(row):].any()


@pytest.mark.parametrize("n", [1, 37, 4001, 262144])
@pytest.mark.parametrize("fs_out", list(RATES))
def test_oracle_matches_resample_poly(fs_out, n):
    """Lengths 1, shorter than every filter here (37), odd (4001) and 262144."""
    up, down = RATES[fs_out]
    x = np.random.default_rng(n).standard_normal(n)
    want = scipy.signal.resample_poly(x, up, down)
    got = resample_ref(x, design_taps(up, down), up, down)
    assert got.shape == want.shape == (-(-n * up // down),)
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def _support_top(rs, j):
    return (j * rs.down + rs.half_len) // rs.up


@pytest.mark.parametrize("chunk_frames", [1, 7, 64, 256])
@pytest.mark.parametrize("fs_out", list(RATES))
def test_emission_tiles_the_output_once(fs_out, chunk_frames):
    """Chunks of chunk_frames * 256 input samples: the emitted ranges tile [0, n_out) exactly once, no output is emitted before the last
    input of its support has arrived (unless the stream ended), and every window's needed inputs lie in the previous and current chunk."""
    rs, hop = Resampler(FS_IN, fs_out), 256
    for frames in (1, 5, 64, 333):
        n, step = frames * hop, chunk_frames * hop
        emitted, prev_start = 0, 0
        for start in range(0, n, step):
            m = min(start + step, n)
            r = rs.ready(m, n, m >= n)
            assert r >= emitted
            if r > emitted and m < n:
                assert _support_top(rs, r - 1) < m and _support_top(rs, r) >= m     # everything ready, nothing early
            if r > emitted:
                lo = max(_support_top(rs, emitted) - rs.K + 1, 0)
                assert lo >= prev_start or step < rs.history
            prev_start, emitted = start, r
        assert emitted == rs.n_out(n)


def test_pool_bookkeeping_with_a_resampler():
    """StreamPool's records for the streams call: previous and current chunk, the stream's length, and contiguous output ranges;
    one chunk per vocoder chunk, ending at n_out."""
    up, chunk = 256, 2
    rs = Resampler(FS_IN, 16000)
    calls = []

    def launch(ptrs, f0s, ns):
        return torch.zeros(len(ptrs), chunk * up)

    def resample(records, max_out):
        calls.append(records)
        return torch.arange(len(records) * max_out, dtype=torch.float32).reshape(len(records), max_out)
    resample.rs = rs
    pool = StreamPool(launch, 80, up, chunk, "cpu", resample=resample)
    ha = pool.add(torch.zeros(80, 5))
    hb = pool.add(torch.zeros(80, 1))
    got = {ha: [], hb: []}
    while len(pool):
        for h, start, y in pool.step():
            got[h].append((start, y.shape[2]))
    for h, n in ((ha, 5), (hb, 1)):
        starts = [s for s, _ in got[h]]
        assert len(got[h]) == -(-n // chunk)
        assert starts[0] == 0 and all(s + w == s2 for (s, w), s2 in zip(got[h], starts[1:]))
        assert sum(w for _, w in got[h]) == rs.n_out(n * up)
    first, second = calls[0], calls[1]
    assert first[0][0] == 0 and first[0][2:6] == (0, 0, chunk * up, 5 * up)                 # no history yet
    assert second[0][2:5] == (0, chunk * up, 2 * chunk * up) and second[0][0] == first[0][1]  # x0 = last step's chunk
    assert second[0][6] == first[0][7]                                                       # outputs continue


@pytest.mark.parametrize("bad", [0, -16000, 16000.5, True, "16000", None])
def test_bad_rates(bad):
    with pytest.raises(ValueError):
        Resampler(FS_IN, bad)
    with pytest.raises(ValueError):
        Resampler(bad, 16000)


def test_ratio_limit():
    assert max(Resampler(FS_IN, 8000).up, Resampler(FS_IN, 8000).down) <= L.RESAMPLE_MAX_FACTOR
    Resampler(2048, 1)                                         # max(up, down) = 2048: accepted
    for a, b in ((22050, 22051), (1, 2049), (48000, 22050 + 1)):
        with pytest.raises(ValueError):
            Resampler(a, b)
    assert Resampler(16000.0, 16000).identity and Resampler(22050, 22050).history == 0


def test_abi_of_the_resampler():
    h = L.lib()
    assert h.fs2_abi_version() == L.ABI_VERSION == 12
    for name in ("fs2_resample", "fs2_resample_window", "fs2_resample_streams"):
        assert hasattr(h, name)
    assert ctypes.sizeof(L.ResampleArgs) == L.RESAMPLE_ARGS_SIZE == 88
    assert ctypes.sizeof(L.ResampleWindowArgs) == L.RESAMPLE_WINDOW_ARGS_SIZE == 144
    assert ctypes.sizeof(L.ResampleStream) == L.RESAMPLE_STREAM_SIZE == 64
    assert ctypes.sizeof(L.ResampleStreamsArgs) == L.RESAMPLE_STREAMS_ARGS_SIZE == 64
    assert [f[0] for f in L.ResampleStream._fields_] == ["x0", "x1", "i0", "i1", "i2", "n", "j0", "j1"]


def _window(**kw):
    rs = Resampler(FS_IN, 16000)
    good = dict(B=2, up=rs.up, down=rs.down, K=rs.K, taps=0x1000, x0=0x1000, x0_batch_stride=512, x1=0x1000, x1_batch_stride=512,
                i0=0, i1=512, i2=1024, N=1024, lens=None, lens_scale=1, j0=0, j1=100, y=0x1000, y_batch_stride=100, pcm16=0,
                scale=32768.0)
    good.update(kw)
    return L.ResampleWindowArgs(**good)


@pytest.mark.parametrize("field,value", [
    ("B", 0), ("up", 0), ("down", -1), ("up", 2049), ("K", 27), ("taps", 0), ("N", 0), ("j0", -1), ("j1", 0), ("j1", 745),
    ("y", 0), ("y_batch_stride", 99), ("i1", 1025), ("x0", 0), ("x1", 0), ("lens_scale", 0), ("i0", 1),
])
def test_window_refusals(field, value):
    """Each bad field alone is FS2_ERR_ARG before any CUDA call (i0 = 1: input 0, which output 0 reads, is not given; j1 = 745 is
    past ceil(1024 * 320 / 441) = 744; lens_scale 0 only matters with lens)."""
    kw = {field: value}
    if field == "lens_scale":
        kw["lens"] = 0x1000
    a = _window(**kw)
    assert L.lib().fs2_resample_window(ctypes.byref(a), None) == -1


def test_window_coverage_rule():
    """Outputs [j0, j1) read inputs [q(j0) - K + 1, q(j1 - 1)] of [0, N): the host refuses a window whose pieces miss the first or the
    last of them (the accepted windows run on the GPU in tests/test_gpu_resample.py)."""
    rs = Resampler(FS_IN, 16000)
    j0, j1 = 200, 300
    lo = (j0 * rs.down + rs.half_len) // rs.up - rs.K + 1
    hi = ((j1 - 1) * rs.down + rs.half_len) // rs.up + 1
    for i0, i2 in ((lo + 1, hi), (lo, hi - 1)):
        a = _window(i0=i0, i1=i0, i2=i2, x0=0, j0=j0, j1=j1, N=10 ** 6, B=1)
        assert L.lib().fs2_resample_window(ctypes.byref(a), None) == -1, (i0, i2)


def test_offline_and_streams_refusals():
    rs = Resampler(FS_IN, 48000)
    h = L.lib()
    good = dict(B=1, up=rs.up, down=rs.down, K=rs.K, taps=0x1000, x=0x1000, x_batch_stride=100, N=100, lens=None, lens_scale=1,
                y=0x1000, y_batch_stride=218, pcm16=0, scale=1.0)
    for k, v in (("x", 0), ("N", 0), ("up", 960), ("down", 294), ("up", 1), ("K", rs.K + 1), ("y", 0)):
        a = L.ResampleArgs(**dict(good, **{k: v}))
        assert h.fs2_resample(ctypes.byref(a), None) == -1, (k, v)
    a = L.ResampleArgs(**dict(good, up=1, down=1, K=21))       # the identity is not a kernel call
    assert h.fs2_resample(ctypes.byref(a), None) == -1
    sgood = dict(B=2, up=rs.up, down=rs.down, K=rs.K, taps=0x1000, table=0x1000, max_out=50, y=0x1000, y_batch_stride=50, pcm16=1,
                 scale=1.0)
    for k, v in (("B", 0), ("table", 0), ("max_out", 0), ("y", 0), ("y_batch_stride", 49), ("K", 0), ("taps", 0)):
        a = L.ResampleStreamsArgs(**dict(sgood, **{k: v}))
        assert h.fs2_resample_streams(ctypes.byref(a), None) == -1, (k, v)
