"""CPU: the streams call's ABI, workspace bound and argument checks (fs2_vocoder_forward_streams), and the StreamPool's bookkeeping
against a substituted launch."""
import ctypes

import pytest
import torch

from fastspeech2_b200 import _lib as L, configs
from fastspeech2_b200.hifigan.models import StreamPool
from tests.test_stream_vocoder_cpu import CONFIGS, _model


def test_abi_of_the_streams_call():
    h = L.lib()
    assert h.fs2_abi_version() == L.ABI_VERSION
    assert ctypes.sizeof(L.VocoderStreamsArgs) == L.VOCODER_STREAMS_ARGS_SIZE == 64
    assert [f[0] for f in L.VocoderStreamsArgs._fields_] == ["B", "frames", "mel", "mel_lens", "f0", "wav", "wav_batch_stride",
                                                            "workspace", "workspace_bytes"]
    for name in ("fs2_vocoder_streams_workspace_bytes", "fs2_vocoder_forward_streams"):
        assert hasattr(h, name)


def _cone(m, frames):
    """conv_pre's input rows [x0, x1) of the unclipped plan of [0, frames): a window far from both ends of a long utterance, shifted."""
    pre = L.vocoder_window_plan(m, 1 << 20, 1000, 1000 + frames)[0]
    assert pre.layer == L.VW_CONV_PRE
    return pre.x0 - 1000, pre.x1 - 1000


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_workspace_is_the_plan_buffers_plus_the_staged_cone_and_tables(cfg):
    """The bound depends on B and frames only, equals the window call's, is the plan's five buffers plus the staged [B][x1 - x0][80]
    mel cone and the [B] origin and length tables, and grows linearly in B."""
    h = L.lib()
    m, _up = _model(CONFIGS[cfg])
    align = lambda n: (n + 255) // 256 * 256           # the workspace arena's alignment of every buffer
    for frames in (1, 7, 32, 64):
        x0, x1 = _cone(m, frames)
        assert x0 < 0 < frames < x1
        width = 0                                      # floats per utterance of each buffer: the widest output of the unclipped plan
        for l in L.vocoder_window_plan(m, 1 << 20, 1000, 1000 + frames)[:-1]:
            ch = m.c0 if l.layer == L.VW_CONV_PRE else (m.c0 >> (l.stage + 1)) * (
                m.rates[l.stage] if l.layer in (L.VW_UP_A, L.VW_UP_B) else 1)
            width = max(width, (l.y1 - l.y0) * ch)
        sizes = []
        for B in (1, 2, 3, 16):
            s = h.fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), B, frames)
            w = h.fs2_vocoder_window_workspace_bytes(ctypes.byref(m), B, frames)
            cone = B * (x1 - x0) * 80 * 4
            assert s == w == 5 * align(4 * B * width) + align(cone) + 2 * align(4 * B) + 256, (frames, B)
            sizes.append(s)
        # linear in B (up to the arena's 256-byte alignment of each of the six buffers)
        per_b = sizes[1] - sizes[0]
        assert abs(sizes[3] - sizes[0] - 15 * per_b) <= 6 * 256 * 16, frames


def test_bad_arguments_are_refused_before_any_cuda_call():
    h = L.lib()
    m, up = _model(configs.HIFIGAN_CONFIG)
    frames = 8
    need = h.fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), 2, frames)
    good = dict(B=2, frames=frames, mel=0x1000, mel_lens=0x1000, f0=0x1000, wav=0x1000, wav_batch_stride=frames * up,
                workspace=0x1000, workspace_bytes=need)
    for k, v in (("B", 0), ("B", -1), ("frames", 0), ("frames", -4), ("mel", 0), ("mel_lens", 0), ("f0", 0), ("wav", 0),
                 ("workspace", 0), ("workspace_bytes", need - 1), ("wav_batch_stride", frames * up - 1)):
        a = L.VocoderStreamsArgs(**dict(good, **{k: v}))
        assert h.fs2_vocoder_forward_streams(ctypes.byref(m), ctypes.byref(a), None) == -1, (k, v)
    assert h.fs2_vocoder_forward_streams(ctypes.byref(m), None, None) == -1
    assert h.fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), 0, frames) == 0
    assert h.fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), 2, 0) == 0


class FakeLaunch:
    """Records each step's table and returns rows that name (stream length, frame, sample) so the chunks can be checked."""

    def __init__(self, up, chunk):
        self.up, self.chunk, self.tables = up, chunk, []

    def __call__(self, ptrs, f0s, ns):
        self.tables.append((list(ptrs), list(f0s), list(ns)))
        i = torch.arange(self.chunk * self.up, dtype=torch.float64)
        return torch.stack([n * 1e6 + f0 * self.up + i for f0, n in zip(f0s, ns)])


def _pool(chunk=3, up=4):
    launch = FakeLaunch(up, chunk)
    return StreamPool(launch, 80, up, chunk, "cpu"), launch


def test_pool_bookkeeping():
    pool, launch = _pool()
    assert pool.step() == [] and launch.tables == []
    mels = {n: torch.randn(80, n) for n in (7, 3, 1, 10)}
    ha = pool.add(mels[7])
    hb = pool.add(mels[3][None])
    assert len(pool) == 2
    s1 = pool.step()
    hc = pool.add(mels[1])                              # joins at frame 0 of the next step
    s2 = pool.step()
    hd = pool.add(mels[10])
    s3 = pool.step()
    s4 = pool.step()
    s5 = pool.step()
    assert [h for h, _, _ in s1] == [ha, hb] and [h for h, _, _ in s2] == [ha, hc] and [h for h, _, _ in s3] == [ha, hd]
    assert [h for h, _, _ in s4] == [hd] and [h for h, _, _ in s5] == [hd] and len(pool) == 1
    assert [t[1] for t in launch.tables] == [[0, 0], [3, 0], [6, 0], [3], [6]]
    assert [t[2] for t in launch.tables] == [[7, 3], [7, 1], [7, 10], [10], [10]]
    # first_sample, the trimmed last chunks and their contents
    up, chunk = 4, 3
    for steps, h, n in ((( s1, s2, s3), ha, 7), ((s1,), hb, 3), ((s2,), hc, 1)):
        first = 0
        for st in steps:
            (start, wav), = [(s, w) for hh, s, w in st if hh == h]
            assert start == first and wav.shape == (1, 1, min(chunk, n - first // up) * up)
            assert torch.equal(wav[0, 0], n * 1e6 + start + torch.arange(wav.shape[2], dtype=torch.float64))
            first += wav.shape[2]
        assert first == n * up
    hd_starts = [s for st in (s3, s4, s5) for hh, s, _ in st if hh == hd]
    assert hd_starts == [0, 12, 24]
    assert pool.step()[0][2].shape == (1, 1, 4) and len(pool) == 0   # frame 9 of 10: trimmed, then the stream leaves


def test_pool_cancel_and_the_uploaded_table():
    pool, launch = _pool(chunk=2)
    rows = torch.randn(3, 9, 80)                        # channels-last, row stride 80: kept without a copy
    hs = [pool.add(rows[b].T) for b in range(3)]
    assert [s[1].data_ptr() for s in pool._live] == [rows[b].data_ptr() for b in range(3)]
    pool.step()
    pool.cancel(hs[1])
    with pytest.raises(KeyError):
        pool.cancel(hs[1])
    pool.step()
    assert launch.tables[-1] == ([rows[0].data_ptr(), rows[2].data_ptr()], [2, 2], [9, 9])
    assert len(pool) == 2


def test_pool_add_checks():
    pool, _ = _pool()
    for bad in (torch.zeros(80, 0), torch.zeros(79, 5), torch.zeros(2, 80, 5), torch.zeros(80), [[0.0] * 5] * 80):
        with pytest.raises(ValueError):
            pool.add(bad)
    odd = torch.randn(5, 80).T[:, ::1].contiguous()      # [80, 5] contiguous: converted to channels-last once
    pool.add(odd)
    kept = pool._live[0][1]
    assert kept.shape == (5, 80) and kept.stride() == (80, 1) and torch.equal(kept, odd.T)
