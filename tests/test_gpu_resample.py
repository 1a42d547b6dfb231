"""GPU: the polyphase resampler (fs2_resample*, resample.Resampler) against the fp64 oracle, and its streamed and pooled forms bit for
bit against the offline call.

Bar of the offline call, per output j: |y - y_ref| <= (K + 3) * 2^-24 * S_j, S_j = sum_i |h[...] * x[i]| over the output's taps.
  - the kernel sums K fused multiply-adds in fp32 (products exact, one rounding each): at most K * 2^-24 * S_j (gamma_K, first order);
  - the taps are fp32 roundings of the fp64 filter: |h32 - h| <= 2^-24 |h|, another 2^-24 * S_j;
  - two more units of slack for the second-order terms.
The inputs are fp32 and enter the oracle exactly."""
import numpy as np
import pytest
import torch

from fastspeech2_b200 import configs, ops, synth
from fastspeech2_b200.resample import Resampler, design_taps
from oracle.resample_ref import resample_ref
from tests.test_gpu_stream_vocoder import _generator

pytestmark = pytest.mark.gpu
DEV = "cuda"
FS_IN = 22050
RATES = (16000, 48000, 24000, 44100, 8000)
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
HOP = 256


def _bar(rs, x):
    h = design_taps(rs.up, rs.down)
    return (rs.K + 3) * 2.0 ** -24 * resample_ref(np.abs(x), np.abs(h), rs.up, rs.down), resample_ref(x, h, rs.up, rs.down)


def _vocoded(B, T, lens, seed):
    gen = _generator(configs.HIFIGAN_CONFIG)
    mel = synth.make_mel(B, T, seed=seed).to(DEV)
    return gen(mel, torch.tensor(lens))                         # [B, 1, T * 256], zeros past lens * 256


@pytest.mark.parametrize("fs_out", RATES)
def test_offline_against_the_oracle(fs_out):
    """B = 3 ragged rows of a strided [B, 1, N] view of Generator output."""
    lens = (48, 31, 7)
    wav = _vocoded(3, 48, lens, seed=1) * 1.25
    N = wav.shape[2]
    buf = torch.full((3, 2, N + 7), float("nan"), device=DEV)
    buf[:, :1, 5:5 + N] = wav
    view = buf[:, :1, 5:5 + N]
    rs = Resampler(FS_IN, fs_out)
    n_samp = torch.tensor(lens) * HOP
    y = rs(view, n_samp)
    assert y.shape == (3, 1, rs.n_out(N)) and y.dtype == torch.float32
    y = y[:, 0].double().cpu().numpy()
    x = wav[:, 0].double().cpu().numpy()
    worst = 0.0
    for b, n in enumerate(n_samp.tolist()):
        bar, ref = _bar(rs, x[b, :n])
        m = rs.n_out(n)
        err = np.abs(y[b, :m] - ref)
        assert (err <= bar + 1e-30).all(), (b, float((err / (bar + 1e-30)).max()))
        assert not y[b, m:].any()
        worst = max(worst, float((err / (bar + 1e-30)).max()))
    print(f"{fs_out} Hz: worst error {worst:.3f} of the bar")


@pytest.mark.parametrize("fs_out", RATES)
def test_ragged_rows_equal_their_solo_calls(fs_out):
    lens = (40, 13, 1)
    wav = _vocoded(3, 40, lens, seed=2)
    rs = Resampler(FS_IN, fs_out)
    y = rs(wav, torch.tensor(lens, device=DEV) * HOP)
    for b, n in enumerate(lens):
        solo = rs(wav[b:b + 1, :, :n * HOP].contiguous())
        m = solo.shape[2]
        assert torch.equal(y[b:b + 1, :, :m], solo) and not y[b, :, m:].any(), b


@pytest.mark.parametrize("fs_out", RATES)
def test_pcm16_equals_wav_to_int16(fs_out):
    wav = _vocoded(2, 30, (30, 19), seed=3) * 8.0                 # past +-1 at every rate: the clamp is reached
    rs = Resampler(FS_IN, fs_out)
    lens = torch.tensor([30, 19]) * HOP
    f = rs(wav[:, 0], lens)
    i = rs(wav[:, 0], lens, pcm16=True, scale=32768.0)
    assert i.dtype == torch.int16 and torch.equal(i, ops.wav_to_int16(f))
    assert int(i.int().abs().max()) >= 32767 and (f.abs() > 1.0).any()    # clamped, not wrapped


def test_identity_returns_the_input():
    wav = _vocoded(2, 10, (10, 4), seed=4)
    rs = Resampler(FS_IN, FS_IN)
    assert rs(wav) is wav
    assert torch.equal(rs(wav, pcm16=True)[:, 0], ops.wav_to_int16(wav[:, 0]))


def test_extreme_ratios_against_the_oracle():
    """max(up, down) = 2048 both ways: the largest tap table (2048 x 21) and a span staged in several passes (up = 1, K = 40961)."""
    x = (torch.rand(1, 2000, generator=torch.Generator().manual_seed(5)) * 2 - 1).to(DEV)
    for fs_in, fs_out in ((1, 2048), (2048, 1), (2047, 2048)):
        rs = Resampler(fs_in, fs_out)
        y = rs(x)[0].double().cpu().numpy()
        bar, ref = _bar(rs, x[0].double().cpu().numpy())
        assert (np.abs(y - ref) <= bar + 1e-30).all(), (fs_in, fs_out)


def _streamed(gen, mel, lens, chunk, rate, pcm16=False):
    parts, first = [], 0
    for start, y in gen.stream(mel, mel_lens=lens, chunk_frames=chunk, sample_rate=rate, pcm16=pcm16):
        assert start == first and y.shape[:2] == (mel.shape[0], 1)
        first += y.shape[2]
        parts.append(y)
    return torch.cat(parts, dim=2), len(parts)


@pytest.mark.parametrize("chunk", [1, 7, 64])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("cfg", list(CFGS))
@pytest.mark.parametrize("fs_out", RATES)
def test_stream_equals_offline(fs_out, cfg, ragged, chunk):
    gen = _generator(CFGS[cfg])
    T, lens = 45, (45, 20, 3)
    mel = synth.make_mel(3, T, seed=6).to(DEV)
    ml = torch.tensor(lens) if ragged else None
    got, n_chunks = _streamed(gen, mel, ml, chunk, fs_out)
    rs = Resampler(FS_IN, fs_out)
    want = rs(gen(mel, ml), None if ml is None else ml * HOP)
    assert n_chunks == -(-T // chunk) and torch.equal(got, want)


def test_stream_pcm16_and_device_lengths():
    gen = _generator(CFGS["v2"])
    mel = synth.make_mel(2, 33, seed=7).to(DEV)
    lens = torch.tensor([33, 12], device=DEV)
    rs = Resampler(FS_IN, 16000)
    got, _ = _streamed(gen, mel, lens, 8, 16000, pcm16=True)
    assert torch.equal(got, rs(gen(mel, lens), lens * HOP, pcm16=True))
    got, _ = _streamed(gen, mel, lens, 8, FS_IN, pcm16=True)    # the generator's own rate
    assert torch.equal(got, ops.wav_to_int16(gen(mel, lens)[:, 0]).unsqueeze(1))
    plain = [y for _, y in gen.stream(mel, lens, chunk_frames=8, sample_rate=FS_IN)]
    assert torch.equal(torch.cat(plain, dim=2), gen(mel, lens))


def _run_pool(pool, mels, join, cancel_at=None, cancel=None):
    """Adds mels[k] before step join[k] (and cancels stream `cancel` before step cancel_at); returns each stream's concatenated
    chunks and chunk count."""
    handles, parts, first = {}, {}, {}
    step = 0
    while step <= max(join) or len(pool):
        for k, j in enumerate(join):
            if j == step:
                handles[k] = pool.add(mels[k])
        if step == cancel_at:
            pool.cancel(handles[cancel])
        for h, start, y in pool.step():
            k = next(k for k, hh in handles.items() if hh == h)
            assert start == first.get(k, 0) and y.dim() == 3 and y.shape[:2] == (1, 1)
            first[k] = start + y.shape[2]
            parts.setdefault(k, []).append(y)
        step += 1
    return {k: (torch.cat(v, dim=2), len(v)) for k, v in parts.items()}


@pytest.mark.parametrize("pcm16", [False, True])
@pytest.mark.parametrize("cfg", list(CFGS))
@pytest.mark.parametrize("fs_out", RATES)
def test_pool_equals_offline(fs_out, cfg, pcm16):
    gen = _generator(CFGS[cfg])
    lens, join = (70, 5, 1, 37, 90), (0, 2, 2, 1, 3)
    mels = [synth.make_mel(1, n, seed=50 + i)[0].to(DEV) for i, n in enumerate(lens)]
    chunk = 16
    got = _run_pool(gen.stream_pool(chunk_frames=chunk, sample_rate=fs_out, pcm16=pcm16), mels, join, cancel_at=3, cancel=0)
    rs = Resampler(FS_IN, fs_out)
    for k, mel in enumerate(mels):
        if k == 0:
            continue                                             # cancelled after three chunks
        y, n_chunks = got[k]
        assert n_chunks == -(-lens[k] // chunk)
        assert torch.equal(y, rs(gen(mel[None]), pcm16=pcm16)), k
    assert got[0][1] == 3


def test_pool_refuses_a_history_longer_than_a_chunk():
    gen = _generator(CFGS["v2"])
    with pytest.raises(ValueError):
        gen.stream_pool(chunk_frames=1, sample_rate=1)          # 22050 -> 1 Hz is refused outright (max(up, down) > 2048)
    with pytest.raises(ValueError):
        gen.stream_pool(chunk_frames=123, sample_rate=14)       # up/down = 1/1575: K - 1 = 31500 > 123 * 256
    with pytest.raises(ValueError):
        gen.stream(synth.make_mel(1, 4).to(DEV), chunk_frames=1, sample_rate=14)
    gen.stream_pool(chunk_frames=124, sample_rate=14)           # 124 * 256 = 31744 >= 31500
