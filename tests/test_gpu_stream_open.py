"""GPU: open streams of the vocoder pool -- mel fed block by block into a fixed ring per stream (StreamPool.open / feed / close,
fs2_mel_ring_append, fs2_vocoder_forward_streams_ring) -- bit for bit against the offline forward of each stream's whole mel.

A chunk joins a step only once its cone has arrived and is computed with n_b = the frames fed so far, which clips nothing inside the
cone, so any difference would show a frame overwritten in the ring before its cone passed, a frame appended to the wrong row, or a
length bound that reached into the cone.  The bar is torch.equal throughout."""
import ctypes

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.hifigan.models import mel_reach
from tests.test_gpu_resample_mixed import _offline
from tests.test_gpu_stream_pool import _streams_call
from tests.test_gpu_stream_vocoder import POLICIES, _generator

pytestmark = pytest.mark.gpu
DEV = "cuda"
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
CHUNK = 32


def _mel(n, seed):
    return synth.make_mel(1, n, seed=seed)[0].to(DEV)


def _blocks(n, pattern, rng):
    """Block sizes that sum to n, and the ticks at which they arrive."""
    if pattern == "one_frame":
        sizes = [1] * n
    elif pattern == "chunk":
        sizes = [CHUNK] * (n // CHUNK) + ([n % CHUNK] if n % CHUNK else [])
    elif pattern == "random":
        sizes = []
        while sum(sizes) < n:
            sizes.append(min(int(rng.integers(1, 60)), n - sum(sizes)))
    elif pattern == "one_block":                       # larger than the ring
        sizes = [n]
    else:                                              # "starved": blocks of 40 with 6 ticks between them
        sizes = [40] * (n // 40) + ([n % 40] if n % 40 else [])
    gap = 6 if pattern == "starved" else 1
    return [(i * gap, m) for i, m in enumerate(sizes)]


def _drive(pool, opened=(), added=()):
    """opened: (mel, open tick, [(tick, block size)], layout) per open stream, closed at its last block's tick; added: (mel, tick) per
    add()ed stream.  Runs the pool to its end and returns each stream's concatenated chunks, checking first_sample."""
    handles, parts, first, fed, rows = {}, {}, {}, {}, {}
    last = max([t0 + b[-1][0] for _, t0, b, _ in opened] + [t for _, t in added] + [0])
    tick = 0
    while tick <= last or len(pool):
        for k, (mel, t0, blocks, layout) in enumerate(opened):
            if tick == t0:
                handles[k] = pool.open()
                fed[k] = 0
                rows[k] = mel.T.contiguous() if layout == "channels_last" else mel.contiguous()
            for t, m in blocks:
                if t0 + t == tick:
                    a = fed[k]
                    pool.feed(handles[k], rows[k][a:a + m].T if layout == "channels_last" else rows[k][:, a:a + m])
                    fed[k] = a + m
            if tick == t0 + blocks[-1][0]:
                pool.close(handles[k])
        for j, (mel, t) in enumerate(added):
            if tick == t:
                handles[("add", j)] = pool.add(mel)
        for h, start, y in pool.step():
            k = next(k for k, v in handles.items() if v == h)
            assert start == first.get(k, 0)
            first[k] = start + y.shape[2]
            parts.setdefault(k, []).append(y)
        tick += 1
    return {k: torch.cat(v, dim=2) for k, v in parts.items()}


@pytest.mark.parametrize("pattern", ["one_frame", "chunk", "random", "one_block", "starved"])
@pytest.mark.parametrize("policy", ["default", "per_layer", "exact"])
@pytest.mark.parametrize("cfg", list(CFGS))
def test_open_stream_equals_forward(cfg, policy, pattern):
    gen = _generator(CFGS[cfg], **POLICIES[policy])
    mel = _mel(301, seed=11)
    got = _drive(gen.stream_pool(chunk_frames=CHUNK), [(mel, 0, _blocks(301, pattern, np.random.default_rng(4)), "channel_major")])
    assert torch.equal(got[0], gen(mel[None]))


@pytest.mark.parametrize("cfg", list(CFGS))
def test_open_and_added_streams_share_the_pool(cfg):
    """Open streams in both layouts and added streams join and leave at other ticks; each equals its forward, and every step makes
    at most one append launch and one vocoder call."""
    gen = _generator(CFGS[cfg])
    rng = np.random.default_rng(9)
    lens = (250, 97, 33, 160)
    mels = [_mel(n, seed=30 + i) for i, n in enumerate(lens)]
    pats = ("random", "one_frame", "one_block", "starved")
    opened = [(mels[k], 3 * k, _blocks(lens[k], pats[k], rng), "channels_last" if k % 2 else "channel_major") for k in range(4)]
    adds = [_mel(n, seed=50 + i) for i, n in enumerate((70, 5, 130))]
    pool = gen.stream_pool(chunk_frames=CHUNK)
    m = gen._packed[0]
    per_call = len(L.vocoder_window_plan(m, 1 << 20, 1000, 1000 + CHUNK)) + 1
    counts = []
    real_step = pool.step

    def step():
        n0 = L.lib().fs2_kernel_launch_count()
        out = real_step()
        counts.append(L.lib().fs2_kernel_launch_count() - n0)
        return out
    pool.step = step
    got = _drive(pool, opened, [(adds[0], 0), (adds[1], 4), (adds[2], 20)])
    torch.cuda.synchronize()
    for k in range(4):
        assert torch.equal(got[k], gen(mels[k][None])), k
    for j in range(3):
        assert torch.equal(got[("add", j)], gen(adds[j][None])), j
    assert set(counts) <= {0, per_call, per_call + 1} and per_call + 1 in counts


@pytest.mark.parametrize("cfg", list(CFGS))
def test_ring_wraps_without_growing(cfg):
    """A 5 000-frame stream through the ring: exact, and its device memory is the ring's whatever its length."""
    gen = _generator(CFGS[cfg])
    mel = _mel(5000, seed=12)
    pool = gen.stream_pool(chunk_frames=CHUNK)
    h = pool.open()
    ring = pool._live[0][1]
    assert ring.shape == (pool.ring_frames, 80) and pool.ring_frames < 100
    parts = []
    for a in range(0, 5000, CHUNK):                    # the pool vocodes a chunk per step: the caller's blocks do not pile up
        pool.feed(h, mel[:, a:a + CHUNK])
        parts += [y for _, _, y in pool.step()]
        assert pool._live[0][1] is ring and sum(b[0].shape[1] - b[1] for b in pool._live[0][8].blocks) <= 2 * CHUNK
    pool.close(h)
    while len(pool):
        parts += [y for _, _, y in pool.step()]
    assert torch.equal(torch.cat(parts, dim=2), gen(mel[None]))
    assert gen.stream_pool(chunk_frames=CHUNK).ring_frames == pool.ring_frames


@pytest.mark.parametrize("cfg", list(CFGS))
def test_open_streams_at_other_rates_and_encodings(cfg):
    gen = _generator(CFGS[cfg])
    rng = np.random.default_rng(6)
    formats = ((8000, "ulaw"), (16000, "pcm16"), (48000, "f32"))
    lens = (180, 77, 241)
    mels = [_mel(n, seed=70 + i) for i, n in enumerate(lens)]
    pool = gen.stream_pool(chunk_frames=CHUNK)
    hs = [pool.open(sample_rate=r, encoding=e) for r, e in formats]
    blocks = [_blocks(n, "random", rng) for n in lens]
    parts, fed = {k: [] for k in range(3)}, [0, 0, 0]
    tick = 0
    while len(pool):
        for k in range(3):
            for t, m in blocks[k]:
                if t == tick:
                    pool.feed(hs[k], mels[k][:, fed[k]:fed[k] + m])
                    fed[k] += m
            if tick == blocks[k][-1][0]:
                pool.close(hs[k])
        for h, _, y in pool.step():
            parts[hs.index(h)].append(y)
        tick += 1
    for k, (rate, enc) in enumerate(formats):
        assert torch.equal(torch.cat(parts[k], dim=2), _offline(gen, mels[k], rate, enc)), formats[k]


def test_append_kernel_equals_copy_into_the_ring():
    gen = _generator(configs.HIFIGAN_V2_CONFIG)
    append = gen.stream_pool(chunk_frames=CHUNK)._append
    cap, fill = 24, -7.0
    rings = [torch.full((cap, 80), fill, device=DEV) for _ in range(4)]
    want = [r.clone() for r in rings]
    src = torch.randn(80, 100, device=DEV)              # channel-major [80, m]
    cl = torch.randn(100, 80, device=DEV)               # channels-last rows; cl[a:b].T is a postnet_mel[b, a:z].T view
    odd = torch.randn(100 * 80 + 1, device=DEV)[1:].view(100, 80)     # channels-last, not 16-byte aligned: scalar loads
    # (tensor [80, m], source frame, ring, destination frame, count): a wrap in both layouts, an unaligned channels-last block whose
    # count is past cap (only its last cap frames remain), and a negative destination frame
    recs = [(src, 3, 0, 17, 20), (cl.T, 5, 1, 40, 12), (odd.T, 0, 2, 0, 30), (src, 60, 3, -5, 9)]
    for t, sf, r, dst, cnt in recs:
        for i in range(cnt):
            want[r][(dst + i) % cap].copy_(t[:, sf + i])
    append([(t.data_ptr(), t.stride(1), t.stride(0), sf, rings[r].data_ptr(), dst, cap, cnt) for t, sf, r, dst, cnt in recs])
    torch.cuda.synchronize()
    for r in range(4):
        assert torch.equal(rings[r], want[r]), r


@pytest.mark.parametrize("cfg", list(CFGS))
def test_ring_call_against_the_streams_call(cfg):
    """cap = n gives the streams call's bits on the same table; a ring holding only the last cap frames written gives them too, and
    cap <= 0 an all-zero chunk."""
    gen = _generator(CFGS[cfg])
    m, _keep, _dev, up = gen._pack()
    frames = 24
    rng = np.random.default_rng(2)
    lens = [int(n) for n in rng.integers(1, 200, size=9)]
    rows = [synth.make_mel(1, n, seed=90 + i)[0].T.contiguous().to(DEV) for i, n in enumerate(lens)]
    f0s = [int(rng.integers(0, n)) for n in lens]
    want = _streams_call(gen, rows, lens, f0s, frames)
    left, right = mel_reach(m, frames)

    def ring_call(ptrs, caps):
        B = len(ptrs)
        tab = torch.tensor(ptrs, dtype=torch.int64, device=DEV)
        lens_d, f0_d, cap_d = (torch.tensor(v, dtype=torch.int32, device=DEV) for v in (lens, f0s, caps))
        need = L.lib().fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), B, frames)
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
        out = torch.full((B, frames * up), float("nan"), device=DEV)
        a = L.VocoderStreamsRingArgs(B=B, frames=frames, mel=tab.data_ptr(), mel_lens=lens_d.data_ptr(), f0=f0_d.data_ptr(),
                                     wav=out.data_ptr(), wav_batch_stride=frames * up, workspace=ws.data_ptr(), workspace_bytes=need,
                                     cap=cap_d.data_ptr())
        L.check(L.lib().fs2_vocoder_forward_streams_ring(ctypes.byref(m), ctypes.byref(a), torch.cuda.current_stream().cuda_stream),
                "ring")
        torch.cuda.synchronize()
        return out
    assert torch.equal(ring_call([r.data_ptr() for r in rows], lens), want)
    cap = left + frames + right
    rings = []
    for r, n, f0 in zip(rows, lens, f0s):
        ring = torch.full((cap, 80), float("nan"), device=DEV)
        top = min(f0 + frames + right, n)               # the frames written so far: the last cap of them are in the ring
        for t in range(max(top - cap, 0), top):
            ring[t % cap] = r[t]
        rings.append(ring)
    assert torch.equal(ring_call([r.data_ptr() for r in rings], [cap] * len(rows)), want)
    caps = [cap] * len(rows)
    caps[3], caps[5] = 0, -4
    got = ring_call([r.data_ptr() for r in rings], caps)
    zero = torch.zeros(frames * up, device=DEV)
    for b in range(len(rows)):
        assert torch.equal(got[b], zero if b in (3, 5) else want[b]), b
