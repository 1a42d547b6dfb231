"""GPU: the windowed vocoder (fs2_vocoder_forward_window, Generator.stream) against the offline forward, bit for bit.

Every window computes its layers' rows from the rows their receptive fields need, in tiles that start at the window, so any
difference from forward would show either a read outside the cone (the NaN poisoning below turns it into NaN) or arithmetic that
depends on a row's position in its tile.  Neither is tolerated: the bar is torch.equal throughout."""
import ctypes
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from tests.test_gpu_ragged_vocoder import POLICIES as RAGGED_POLICIES

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
T = 90
LENS = (90, 5, 0)                                        # full, shorter than the first chunk, empty
POLICIES = {
    "default": {},
    "pairs": {"fused_mask": 0},                           # V1 / V2: the pair_mask stages run fused pairs
    "per_layer": {"fused_mask": 0, "pair_mask": 0},
    "exact": {"use_tensor_cores": False},
}


def _generator(cfg, seed=3, sd=None, **policy):
    h = AttrDict(cfg)
    gen = Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=seed) if sd is None else sd)
    gen.eval()
    gen.remove_weight_norm()
    for k, v in policy.items():
        setattr(gen, k, v)
    gen._invalidate()
    return gen.to(DEV)


def _postnet_view(B, frames, seed):
    """A strided postnet_mel.transpose(1, 2) view, as FastSpeech2's caller passes it."""
    return synth.make_mel(B, frames, seed=seed).transpose(1, 2).contiguous().to(DEV).transpose(1, 2)


def _streamed(gen, mel, lens, chunk):
    parts, first = [], 0
    for start, wav in gen.stream(mel, mel_lens=lens, chunk_frames=chunk):
        assert start == first and wav.shape[:2] == (mel.shape[0], 1)
        first += wav.shape[2]
        parts.append(wav)
    return torch.cat(parts, dim=2)


@pytest.mark.parametrize("chunk", [1, 7, 64, 200])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("cfg", ["v1", "v2"])
def test_stream_equals_forward(cfg, policy, ragged, chunk):
    gen = _generator(configs.HIFIGAN_CONFIG if cfg == "v1" else configs.HIFIGAN_V2_CONFIG, **POLICIES[policy])
    mel = _postnet_view(len(LENS), T, seed=21)
    lens = torch.tensor(LENS) if ragged else None
    want = gen(mel, lens)
    got = _streamed(gen, mel, lens, chunk)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("policy", list(RAGGED_POLICIES) + ["wide_pairs"])
@pytest.mark.parametrize("cfg", ["v1", "v2"])
def test_forward_launches_the_plan_of_the_whole_batch(cfg, policy, ragged):
    """forward issues fs2_vocoder_window_plan(m, T, 0, T): one kernel per record."""
    gen = _generator(configs.HIFIGAN_CONFIG if cfg == "v1" else configs.HIFIGAN_V2_CONFIG,
                     **({"wide_pairs": True} if policy == "wide_pairs" else RAGGED_POLICIES[policy]))
    mel = _postnet_view(len(LENS), T, seed=22)          # a channels-last view: forward launches no transpose
    lens = torch.tensor(LENS) if ragged else None
    gen(mel, lens)                                      # packs the weights
    torch.cuda.synchronize()
    n0 = L.lib().fs2_kernel_launch_count()
    gen(mel, lens)
    launches = L.lib().fs2_kernel_launch_count() - n0
    assert launches == len(L.vocoder_window_plan(gen._packed[0], T, 0, T))


def test_stream_contiguous_mel_and_lengths_on_the_device():
    gen = _generator(configs.HIFIGAN_CONFIG)
    mel = synth.make_mel(3, 50, seed=22).to(DEV)
    lens = torch.tensor([50, 17, 33], device=DEV)
    assert torch.equal(_streamed(gen, mel, lens, 16), gen(mel, lens))


def test_stream_argument_checks():
    gen = _generator(configs.HIFIGAN_V2_CONFIG)
    mel = synth.make_mel(2, 20, seed=23).to(DEV)
    for bad in (torch.tensor([21, 3]), torch.tensor([-1, 3]), torch.tensor([3.0, 4.0]), torch.tensor([3])):
        with pytest.raises(ValueError):
            gen.stream(mel, mel_lens=bad)
    for chunk in (0, -3, 2.5, True):
        with pytest.raises(ValueError):
            gen.stream(mel, chunk_frames=chunk)
    with pytest.raises(ValueError):
        gen.stream(mel[:, :40])


def _window_call(gen, mel_cl, lens_d, f0, f1, out, out_bs, ws):
    m, _keep, _dev, _up = gen._packed or gen._pack()
    B, Tm, _ = mel_cl.shape
    a = L.VocoderWindowArgs(B=B, T=Tm, mel=mel_cl.data_ptr(), mel_batch_stride=mel_cl.stride(0), mel_row_stride=mel_cl.stride(1),
                            wav=out.data_ptr(), workspace=ws.data_ptr(), workspace_bytes=ws.numel() * ws.element_size(), mel_lens=L.ptr(lens_d),
                            f0=f0, f1=f1, wav_batch_stride=out_bs)
    L.check(L.lib().fs2_vocoder_forward_window(ctypes.byref(m), ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "window")


@pytest.mark.parametrize("ragged", [False, True, "clamped"])
@pytest.mark.parametrize("cfg", ["v1", "v2"])
def test_windows_in_reverse_order_into_the_full_waveform(cfg, ragged):
    """Stateless windows, written straight into a preallocated waveform at sample f0 * up (wav_batch_stride = T * up), last first
    and the first one twice.  clamped: device lengths outside [0, T], read as clamped to it, and mel rows 84 floats apart (forward
    runs conv_pre on the fp32 kernel for that layout, and so must the window)."""
    gen = _generator(configs.HIFIGAN_CONFIG if cfg == "v1" else configs.HIFIGAN_V2_CONFIG)
    m, _keep, _dev, up = gen._pack()
    mel = _postnet_view(len(LENS), T, seed=24)
    lens_d = torch.tensor(LENS, dtype=torch.int32, device=DEV) if ragged else None
    want = gen(mel, lens_d)
    if ragged == "clamped":
        wide = torch.full((len(LENS), T, 84), NAN, device=DEV)
        wide[:, :, :80] = mel.transpose(1, 2)
        mel = wide[:, :, :80].transpose(1, 2)
        lens_d = torch.tensor((T + 7, -3, 40), dtype=torch.int32, device=DEV)
        want = gen(mel, torch.tensor((T, 0, 40)))
    mel_cl = mel.transpose(1, 2)
    chunk = 13
    ws = torch.empty(L.lib().fs2_vocoder_window_workspace_bytes(ctypes.byref(m), len(LENS), chunk), dtype=torch.uint8, device=DEV)
    full = torch.full_like(want, NAN)
    for f0 in list(range(0, T, chunk))[::-1] + [0]:
        _window_call(gen, mel_cl, lens_d, f0, f0 + chunk, full[:, 0, f0 * up:], T * up, ws)
    torch.cuda.synchronize()
    assert torch.equal(full, want)


@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("cfg", ["v1", "v2"])
def test_reads_stay_inside_the_cone(cfg, ragged, policy):
    """The workspace and every mel row outside the window's cone (conv_pre's input rows of the plan), or at or past n_b, are NaN."""
    gen = _generator(configs.HIFIGAN_CONFIG if cfg == "v1" else configs.HIFIGAN_V2_CONFIG, **POLICIES[policy])
    m, _keep, _dev, up = gen._pack()
    mel = synth.make_mel(len(LENS), T, seed=25).to(DEV)
    lens = (90, 40, 0)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV) if ragged else None
    want = gen(mel, lens_d)
    for f0, f1 in ((0, 7), (33, 61), (80, 120), (45, 46)):
        pre = L.vocoder_window_plan(m, T, f0, f1)[0]
        poisoned = torch.full((len(LENS), T, 80), NAN, device=DEV)
        for b, n in enumerate(lens):
            hi = min(pre.x1, n) if ragged else pre.x1
            if hi > pre.x0:
                poisoned[b, pre.x0:hi] = mel[b, :, pre.x0:hi].T
        ws = torch.full((L.lib().fs2_vocoder_window_workspace_bytes(ctypes.byref(m), len(LENS), f1 - f0) // 4,), NAN, device=DEV)
        n = (min(f1, T) - f0) * up
        out = torch.full((len(LENS), n), NAN, device=DEV)
        _window_call(gen, poisoned, lens_d, f0, f1, out, n, ws)
        torch.cuda.synchronize()
        assert torch.equal(out, want[:, 0, f0 * up:min(f1, T) * up]), (f0, f1)


def test_long_utterance_in_bounded_workspace():
    """A 20 000-frame utterance in 64-frame chunks: the same waveform as forward, in a workspace below 1/50 of forward's."""
    gen = _generator(configs.HIFIGAN_CONFIG)
    m, _keep, _dev, _up = gen._pack()
    frames = 20000
    mel = synth.make_mel(1, frames, seed=26).to(DEV)
    want = gen(mel)
    got = _streamed(gen, mel, None, 64)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    h = L.lib()
    assert h.fs2_vocoder_window_workspace_bytes(ctypes.byref(m), 1, 64) * 50 < h.fs2_vocoder_workspace_bytes(ctypes.byref(m), 1, frames)


def test_chunk_longer_than_the_batch():
    gen = _generator(configs.HIFIGAN_V2_CONFIG)
    mel = _postnet_view(2, 40, seed=27)
    chunks = list(gen.stream(mel, chunk_frames=500))
    assert len(chunks) == 1 and chunks[0][0] == 0 and torch.equal(chunks[0][1], gen(mel))


@pytest.mark.parametrize("name", ["LJSpeech", "universal"])
def test_stream_real_checkpoint(name):
    from oracle import real_ckpt
    sd = real_ckpt.load(name)
    if sd is None:
        pytest.skip("oracle/_ref/ real-checkpoint fixture not in this snapshot")
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"hifigan_real_{name}.npz"))
    gold = torch.from_numpy(z["mel"])[:1]
    Tg = gold.shape[2]
    mel = torch.zeros(3, 80, Tg)
    lens = (Tg, Tg // 2, 3)
    for b, n in enumerate(lens):
        mel[b, :, :n] = gold[0, :, :n]
    gen = _generator(configs.HIFIGAN_CONFIG, sd=sd)
    mel = mel.to(DEV)
    for ragged in (False, True):
        ml = torch.tensor(lens) if ragged else None
        assert torch.equal(_streamed(gen, mel, ml, 64), gen(mel, ml)), ragged
