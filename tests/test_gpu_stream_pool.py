"""GPU: many streams at their own positions in one call (fs2_vocoder_forward_streams, Generator.stream_pool), bit for bit against the
offline forward of each stream alone.

Every kernel bounds each utterance by its own origin, so any difference would show a read outside a stream's cone (the NaN poisoning
turns it into NaN), a dependence on the other streams of the call, or arithmetic that depends on where a row sits in its tile.  None
is tolerated: the bar is torch.equal throughout."""
import ctypes
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from tests.test_gpu_stream_vocoder import POLICIES, _generator

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
LENS = (90, 5, 1, 37, 200)
JOIN = (0, 2, 2, 1, 3)                                   # the step before which each stream is added
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}


def _mels(lens, seed):
    return [synth.make_mel(1, n, seed=seed + i)[0].to(DEV) for i, n in enumerate(lens)]


def _run_pool(pool, mels, join):
    """Adds mels[k] before step join[k]; returns each stream's concatenated chunks, checking first_sample and the chunk widths."""
    handles, parts, first = {}, {}, {}
    step = 0
    while step <= max(join, default=-1) or len(pool):
        for k, j in enumerate(join):
            if j == step:
                handles[pool.add(mels[k])] = k
        for h, start, wav in pool.step():
            k = handles[h]
            assert start == first.get(k, 0) and wav.dim() == 3 and wav.shape[:2] == (1, 1)
            assert wav.shape[2] <= pool.chunk_frames * pool.up
            first[k] = start + wav.shape[2]
            parts.setdefault(k, []).append(wav)
        step += 1
    return {k: torch.cat(v, dim=2) for k, v in parts.items()}


@pytest.mark.parametrize("chunk", [1, 7, 64])
@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("cfg", list(CFGS))
def test_pool_equals_forward(cfg, policy, chunk):
    gen = _generator(CFGS[cfg], **POLICIES[policy])
    mels = _mels(LENS, seed=40)
    got = _run_pool(gen.stream_pool(chunk_frames=chunk), mels, JOIN)
    torch.cuda.synchronize()
    for k, mel in enumerate(mels):
        assert torch.equal(got[k], gen(mel[None])), (k, LENS[k])


def _streams_call(gen, rows, lens, f0s, frames, ws=None):
    """One fs2_vocoder_forward_streams call: rows[b] is stream b's [>= 1, 80] channels-last mel, lens[b] its n_b."""
    m, _keep, _dev, up = gen._packed or gen._pack()
    B = len(rows)
    ptrs = torch.tensor([r.data_ptr() for r in rows], dtype=torch.int64, device=DEV)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    f0_d = torch.tensor(f0s, dtype=torch.int32, device=DEV)
    need = L.lib().fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), B, frames)
    if ws is None:
        ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    assert ws.numel() * ws.element_size() >= need
    out = torch.full((B, frames * up), NAN, device=DEV)
    a = L.VocoderStreamsArgs(B=B, frames=frames, mel=ptrs.data_ptr(), mel_lens=lens_d.data_ptr(), f0=f0_d.data_ptr(), wav=out.data_ptr(),
                             wav_batch_stride=frames * up, workspace=ws.data_ptr(), workspace_bytes=ws.numel() * ws.element_size())
    L.check(L.lib().fs2_vocoder_forward_streams(ctypes.byref(m), ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "streams")
    torch.cuda.synchronize()
    return out


def _expected(full, f0, frames, up):
    """forward's samples [f0 * up, (f0 + frames) * up) of one stream, zeros outside [0, n * up)."""
    out = torch.zeros(frames * up, device=DEV)
    lo, hi = f0 * up, (f0 + frames) * up
    a, b = max(lo, 0), min(hi, full.numel())
    if b > a:
        out[a - lo:b - lo] = full[a:b]
    return out


@pytest.mark.parametrize("cfg", list(CFGS))
def test_batch_invariance(cfg):
    """The same (stream, f0) alone and among 40 neighbours at other offsets, ended streams, n_b = 0 and a negative f0 among them."""
    gen = _generator(CFGS[cfg])
    up = gen._pack()[3]
    frames = 24
    rng = np.random.default_rng(5)
    lens = [int(n) for n in rng.integers(1, 160, size=41)]
    lens[0] = 150
    lens[7] = 0
    rows = [synth.make_mel(1, max(n, 1), seed=60 + i)[0].T.contiguous().to(DEV) for i, n in enumerate(lens)]
    f0s = [int(f) for f in rng.integers(0, 140, size=41)]
    f0s[0] = 61
    f0s[3] = lens[3] + 5                                 # ended
    f0s[9] = -10                                         # before the utterance
    alone = _streams_call(gen, rows[:1], lens[:1], f0s[:1], frames)
    crowd = _streams_call(gen, rows, lens, f0s, frames)
    assert torch.equal(alone[0], crowd[0])
    for b in (0, 3, 7, 9, 20):
        full = gen(rows[b].T[None, :, :max(lens[b], 1)])[0, 0] if lens[b] > 0 else torch.zeros(0, device=DEV)
        assert torch.equal(crowd[b], _expected(full, f0s[b], frames, up)), b


@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("cfg", list(CFGS))
def test_reads_stay_inside_the_cone(cfg, policy):
    """Each stream's mel rows outside its cone (conv_pre's input rows of the unclipped plan, shifted by f0) or at or past n_b are NaN,
    and so is the workspace."""
    gen = _generator(CFGS[cfg], **POLICIES[policy])
    m, _keep, _dev, up = gen._pack()
    frames = 16
    pre = L.vocoder_window_plan(m, 1 << 20, 1000, 1000 + frames)[0]
    x0, x1 = pre.x0 - 1000, pre.x1 - 1000
    lens, f0s = (90, 40, 8, 60), (33, 30, 0, 59)
    mels = _mels(lens, seed=70)
    rows = []
    for mel, n, f0 in zip(mels, lens, f0s):
        r = torch.full((n + 20, 80), NAN, device=DEV)
        lo, hi = max(f0 + x0, 0), min(f0 + x1, n)
        if hi > lo:
            r[lo:hi] = mel[:, lo:hi].T
        rows.append(r)
    need = L.lib().fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), len(rows), frames)
    ws = torch.full((need // 4 + 1,), NAN, device=DEV)
    out = _streams_call(gen, rows, lens, f0s, frames, ws)
    for b, mel in enumerate(mels):
        assert torch.equal(out[b], _expected(gen(mel[None])[0, 0], f0s[b], frames, up)), b


@pytest.mark.parametrize("cfg", list(CFGS))
def test_window_and_streams_calls_launch_the_plan_plus_staging(cfg):
    """One call: the launches of the plan of its frames plus the staging launch, whatever B is, as a fs2_vocoder_forward_window of
    the same frames issues."""
    gen = _generator(CFGS[cfg])
    m, _keep, _dev, up = gen._pack()
    frames = 32
    h = L.lib()
    mel = synth.make_mel(1, 100, seed=80).to(DEV)
    chunks = gen.stream(mel, chunk_frames=frames)      # converts the mel when called
    n0 = h.fs2_kernel_launch_count()
    next(chunks)
    window = h.fs2_kernel_launch_count() - n0
    assert window == len(L.vocoder_window_plan(m, 100, 0, frames)) + 1
    rows = [mel[0].T.contiguous()] * 17
    for B in (1, 17):
        n0 = h.fs2_kernel_launch_count()
        _streams_call(gen, rows[:B], [100] * B, [i * 5 for i in range(B)], frames)
        assert h.fs2_kernel_launch_count() - n0 == window, B


def test_mel_layouts_give_the_same_bits():
    """FastSpeech2's postnet_mel[b, :n].T (kept without a copy) and a contiguous [80, n]."""
    gen = _generator(configs.HIFIGAN_CONFIG)
    postnet = synth.make_mel(2, 70, seed=90).transpose(1, 2).contiguous().to(DEV)   # [B, T, 80]
    views = [postnet[0, :70].T, postnet[1, :45].T]
    pool = gen.stream_pool(chunk_frames=16)
    for v in views:
        pool.add(v)
    assert all(s[1].data_ptr() == v.data_ptr() for s, v in zip(pool._live, views))   # no copy
    a = _run_pool(gen.stream_pool(chunk_frames=16), views, (0, 0))
    pool_b = _run_pool(gen.stream_pool(chunk_frames=16), [v.contiguous() for v in views], (0, 0))
    for k in (0, 1):
        assert torch.equal(a[k], pool_b[k]) and torch.equal(a[k], gen(views[k].contiguous()[None])), k


def test_pool_argument_checks():
    gen = _generator(configs.HIFIGAN_V2_CONFIG)
    pool = gen.stream_pool(chunk_frames=8)
    n0 = L.lib().fs2_kernel_launch_count()
    assert pool.step() == [] and len(pool) == 0
    assert L.lib().fs2_kernel_launch_count() == n0
    for bad in (torch.zeros(80, 0, device=DEV), torch.zeros(79, 10, device=DEV), torch.zeros(2, 80, 10, device=DEV),
                torch.zeros(80, 10)):
        with pytest.raises(ValueError):
            pool.add(bad)
    for chunk in (0, -1, 1.5, True):
        with pytest.raises(ValueError):
            gen.stream_pool(chunk_frames=chunk)
    h = pool.add(torch.zeros(1, 80, 30, device=DEV))
    assert len(pool) == 1
    pool.cancel(h)
    assert len(pool) == 0 and pool.step() == []
    with pytest.raises(KeyError):
        pool.cancel(h)


@pytest.mark.parametrize("name", ["LJSpeech", "universal"])
def test_pool_real_checkpoint(name):
    from oracle import real_ckpt
    sd = real_ckpt.load(name)
    if sd is None:
        pytest.skip("oracle/_ref/ real-checkpoint fixture not in this snapshot")
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"hifigan_real_{name}.npz"))
    gold = torch.from_numpy(z["mel"])[0].to(DEV)
    Tg = gold.shape[1]
    mels = [gold, gold[:, :Tg // 2].contiguous(), gold[:, :3].contiguous()]
    gen = _generator(configs.HIFIGAN_CONFIG, sd=sd)
    got = _run_pool(gen.stream_pool(chunk_frames=64), mels, (0, 1, 1))
    for k, mel in enumerate(mels):
        assert torch.equal(got[k], gen(mel[None])), k
