"""CPU: open streams of the vocoder pool -- the ring call's and the append call's ABI against the C header and their argument checks
(fs2_vocoder_forward_streams_ring, fs2_mel_ring_append), mel_reach against the plan, and StreamPool's readiness, ring and block
bookkeeping against a substituted launch and append."""
import ctypes
import os
import re
import weakref

import pytest
import torch

from fastspeech2_b200 import _lib as L, configs
from fastspeech2_b200.hifigan.models import StreamPool, mel_reach
from fastspeech2_b200.resample import Resampler
from tests.test_stream_vocoder_cpu import CONFIGS, _model

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "fs2b200.h")
C_SIZES = {"int": 4, "int32_t": 4, "int64_t": 8, "size_t": 8, "float": 4}


def _c_layout(name):
    """[(field, offset)] and sizeof of `typedef struct name {...}` in the header, by the x86-64 rules: every field naturally aligned
    (pointers 8 bytes), the size rounded up to the largest alignment."""
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), open(HEADER).read(), re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    out, off, align = [], 0, 1
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        decl = re.sub(r"\bconst\b", "", decl)
        base = re.match(r"\s*(\w+)", decl).group(1)
        for var in decl[decl.index(base) + len(base):].split(","):
            size = 8 if "*" in var else C_SIZES[base]
            off = -(-off // size) * size
            out.append((var.replace("*", "").strip(), off))
            off += size
            align = max(align, size)
    return out, -(-off // align) * align


@pytest.mark.parametrize("cname,cls,size", [("fs2_vocoder_streams_ring_args", L.VocoderStreamsRingArgs, 72),
                                            ("fs2_mel_ring_record_t", L.MelRingRecord, 56),
                                            ("fs2_mel_ring_append_args", L.MelRingAppendArgs, 24)])
def test_abi_against_the_header(cname, cls, size):
    fields, csize = _c_layout(cname)
    assert csize == ctypes.sizeof(cls) == size
    assert fields == [(n, getattr(cls, n).offset) for n, _ in cls._fields_]
    h = L.lib()
    assert h.fs2_abi_version() == L.ABI_VERSION
    for name in ("fs2_vocoder_forward_streams_ring", "fs2_mel_ring_append"):
        assert hasattr(h, name)


def test_ring_call_refuses_bad_arguments_before_any_cuda_call():
    h = L.lib()
    m, up = _model(configs.HIFIGAN_CONFIG)
    frames = 8
    need = h.fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), 2, frames)
    good = dict(B=2, frames=frames, mel=0x1000, mel_lens=0x1000, f0=0x1000, wav=0x1000, wav_batch_stride=frames * up,
                workspace=0x1000, workspace_bytes=need, cap=0x1000)
    for k, v in (("B", 0), ("B", -1), ("frames", 0), ("mel", 0), ("mel_lens", 0), ("f0", 0), ("cap", 0), ("wav", 0),
                 ("workspace", 0), ("workspace_bytes", need - 1), ("wav_batch_stride", frames * up - 1)):
        a = L.VocoderStreamsRingArgs(**dict(good, **{k: v}))
        assert h.fs2_vocoder_forward_streams_ring(ctypes.byref(m), ctypes.byref(a), None) == -1, (k, v)
    assert h.fs2_vocoder_forward_streams_ring(ctypes.byref(m), None, None) == -1


def test_append_call_refuses_bad_arguments_before_any_cuda_call():
    h = L.lib()
    good = dict(table=0x1000, n_records=3, n_mel=80, max_count=8)
    for k, v, rc in (("table", 0, -1), ("n_records", 0, -1), ("n_records", -2, -1), ("max_count", 0, -1), ("max_count", -1, -1),
                     ("n_mel", 0, -2), ("n_mel", 78, -2)):
        a = L.MelRingAppendArgs(**dict(good, **{k: v}))
        assert h.fs2_mel_ring_append(ctypes.byref(a), None) == rc, (k, v)
    assert h.fs2_mel_ring_append(None, None) == -1


@pytest.mark.parametrize("cfg", ["v1", "v2"])
def test_reach_is_the_conv_pre_record_of_an_unclipped_window(cfg):
    m, _up = _model(CONFIGS[cfg])
    for chunk in (1, 8, 32, 64, 100):
        left, right = mel_reach(m, chunk)
        for f0 in (500, 3001):
            pre = L.vocoder_window_plan(m, 20000, f0, f0 + chunk)[0]
            assert pre.layer == L.VW_CONV_PRE
            assert (pre.x0, pre.x1) == (f0 - left, f0 + chunk + right), (chunk, f0)
        assert left > 0 and right > 0


# ------------------------------------------------------------------ the pool against a substituted launch and append
REACH, CHUNK, UP = (5, 4), 3, 2


class Device:
    """Stands in for the device: rings as {row: stream frame}, and the blocks fed as their first stream frame.  The launch checks that
    every frame of each ring stream's cone is in its ring, and returns rows naming (n, sample) as FakeLaunch in test_stream_pool_cpu."""

    def __init__(self, chunk=CHUNK):
        self.chunk, self.rings, self.blocks, self.calls, self.appends = chunk, {}, {}, [], []

    def block(self, t, first):
        self.blocks[t.data_ptr()] = (t.shape[1], t.stride(), first)    # no reference: the pool alone keeps the block alive
        return t

    def append(self, records):
        self.calls.append("append")
        self.appends.append(list(records))
        rows = set()
        for src, fs, cs, sf, ring, dst, cap, count in records:
            m, stride, first = self.blocks[src]
            assert (fs, cs) == (stride[1], stride[0]) and 0 <= sf and sf + count <= m
            assert first + sf == dst and 0 < count <= cap
            for i in range(count):
                assert (ring, (dst + i) % cap) not in rows    # one launch never writes a ring row twice
                rows.add((ring, (dst + i) % cap))
                self.rings.setdefault(ring, {})[(dst + i) % cap] = dst + i

    def launch(self, ptrs, f0s, ns, caps=None):
        self.calls.append("launch" if caps is None else "ring")
        self.last = (list(ptrs), list(f0s), list(ns), caps and list(caps))
        if caps is not None:
            for p, f0, n, cap in zip(ptrs, f0s, ns, caps):
                if p in self.rings:
                    ring = self.rings[p]
                    for t in range(max(f0 - REACH[0], 0), min(f0 + self.chunk + REACH[1], n)):
                        assert ring.get(t % cap) == t, (t, f0, n)
                else:
                    assert cap == n
        i = torch.arange(self.chunk * UP, dtype=torch.float64)
        return torch.stack([n * 1e6 + f0 * UP + i for f0, n in zip(f0s, ns)])


def _pool(**kw):
    dev = Device()
    return StreamPool(dev.launch, 80, UP, CHUNK, "cpu", append=dev.append, reach=REACH, **kw), dev


def _feed(pool, dev, h, m, fed, layout="channel_major"):
    t = torch.randn(80, m) if layout == "channel_major" else torch.randn(m + 2, 80)[1:m + 1].T
    pool.feed(h, dev.block(t, fed))
    return fed + m


def test_readiness_joined_set_and_lengths():
    pool, dev = _pool()
    assert pool.ring_frames == 16                       # 5 + 3 + 4 rounded up to 8
    a = pool.open()
    assert pool.step() == [] and dev.calls == []         # nothing fed: no call at all
    fed = _feed(pool, dev, a, 6, 0)
    assert pool.step() == [] and dev.calls == []         # 6 < 0 + 3 + 4
    fed = _feed(pool, dev, a, 1, fed, "channels_last")
    hb = pool.add(torch.randn(80, 4))
    out = pool.step()                                    # a: 7 >= 7 joins with n = 7; b rides in the ring call as cap = n
    assert [h for h, _, _ in out] == [a, hb] and dev.calls == ["append", "ring"]
    assert dev.last[1:] == ([0, 0], [7, 4], [16, 4])
    assert [w.shape[2] for _, _, w in out] == [CHUNK * UP, CHUNK * UP]
    out = pool.step()                                    # a starves (needs 10), b goes on alone on the plain call
    assert [h for h, _, _ in out] == [hb] and dev.calls[-1] == "launch" and dev.last[1:] == ([3], [4], None)
    assert pool.step() == [] and len(pool) == 1          # b has left; a waits
    fed = _feed(pool, dev, a, 20, fed)
    starts = []
    for _ in range(6):
        out = pool.step()
        assert [h for h, _, _ in out] == [a]
        starts.append(out[0][1])
        assert dev.last[2] == [fed]
    assert starts == [3 * UP, 6 * UP, 9 * UP, 12 * UP, 15 * UP, 18 * UP]
    assert pool.step() == []                             # [21, 24) needs 21 + 3 + 4 = 28 > 27 frames
    pool.close(a)
    tail = []
    while len(pool):
        out = pool.step()
        assert dev.last[2] == [27] and dev.last[3] == [16]
        tail += [(s, w.shape[2]) for _, s, w in out]
    assert tail == [(21 * UP, 3 * UP), (24 * UP, 3 * UP)]


def test_a_large_block_is_drained_over_several_steps_and_then_released():
    pool, dev = _pool()
    a = pool.open()
    big = dev.block(torch.randn(1000, 80).T, 0)          # a channels-last view, kept without a copy
    ref = weakref.ref(big)
    pool.feed(a, big)
    del big
    n_steps = 0
    while ref() is not None:
        out = pool.step()
        n_steps += 1
        assert len(out) == 1 and dev.calls[-2:] == ["append", "ring"]
        counts = [r[7] for r in dev.appends[-1]]
        assert counts == ([CHUNK + REACH[1]] if n_steps == 1 else [CHUNK])
        assert pool._live[0][1].shape == (pool.ring_frames, 80)
    assert pool._live[0][8].written == 1000 and not pool._live[0][8].blocks
    pool.close(a)
    while len(pool):
        pool.step()
    assert n_steps == (1000 - CHUNK - REACH[1]) // CHUNK + 1


def test_many_streams_share_the_append_call():
    """Open streams fed in other block sizes, starved, closed and added ones joining at other steps: every step makes at most one
    append call and one launch, and every stream's chunks tile its frames."""
    pool, dev = _pool()
    sizes = {0: [1] * 40, 1: [7, 1, 30], 2: [13] * 3, 3: [2, 50]}
    fed, hs, added = {}, {}, {}
    got = {}
    for tick in range(80):
        if tick < 4:
            hs[tick] = pool.open()
            fed[tick] = 0
        if tick in (3, 9):
            added[pool.add(torch.randn(80, 11 + tick))] = 11 + tick
        for k, blocks in sizes.items():
            if k in hs and blocks and tick % (k + 1) == 0:
                fed[k] = _feed(pool, dev, hs[k], blocks.pop(0), fed[k], "channels_last" if k % 2 else "channel_major")
                if not blocks:
                    pool.close(hs[k])
        before = len(dev.calls)
        for h, s, w in pool.step():
            got.setdefault(h, []).append((s, w.shape[2]))
        assert dev.calls[before:] in ([], ["launch"], ["ring"], ["append", "ring"])
    assert len(pool) == 0
    total = {**added, **{hs[k]: fed[k] for k in hs}}
    for h, parts in got.items():
        assert [s for s, _ in parts] == [i * CHUNK * UP for i in range(len(parts))]
        assert sum(w for _, w in parts) == total[h] * UP, h


def test_open_feed_close_errors():
    pool, dev = _pool()
    with pytest.raises(ValueError):
        StreamPool(dev.launch, 80, UP, CHUNK, "cpu").open()            # no append call
    a = pool.open()
    for bad in (torch.zeros(80, 0), torch.zeros(79, 5), torch.zeros(2, 80, 5), torch.zeros(80), torch.zeros(80, 5, dtype=torch.int32),
                torch.zeros(80, 5, device="meta"), [[0.0] * 5] * 80):
        with pytest.raises(ValueError):
            pool.feed(a, bad)
    pool.feed(a, torch.zeros(1, 80, 2, dtype=torch.float64))          # another float type: converted once
    assert pool._live[0][8].blocks[0][0].dtype == torch.float32
    with pytest.raises(KeyError):
        pool.feed(a + 100, torch.zeros(80, 2))
    with pytest.raises(KeyError):
        pool.close(a + 100)
    hb = pool.add(torch.zeros(80, 4))
    with pytest.raises(ValueError):
        pool.feed(hb, torch.zeros(80, 2))
    with pytest.raises(ValueError):
        pool.close(hb)
    pool.close(a)
    with pytest.raises(ValueError):
        pool.feed(a, torch.zeros(80, 2))
    with pytest.raises(ValueError):
        pool.close(a)
    e = pool.open()
    pool.close(e)                                        # closed with no frames: leaves without output
    assert [s[0] for s in pool._live] == [a, hb]
    with pytest.raises(KeyError):
        pool.feed(e, torch.zeros(80, 2))


def test_ready_of_a_stream_of_unknown_length():
    for fs_out in (8000, 16000, 22050, 48000):
        rs = Resampler(22050, fs_out)
        for m in (0, 1, 100, 5000):
            assert rs.ready(m, None, False) == rs.ready(m, 10 ** 9, False)


def test_conversion_of_an_open_stream_emits_the_whole_output_once():
    """An open stream at another rate: each step's records ask for the outputs that became ready, contiguous, and the last, after
    close, flushes up to n_out of the stream's samples."""
    seen = []

    def resample(records, max_out):
        seen.extend(records)
        return torch.zeros(len(records), max(max_out, 1))
    resample.rs = Resampler(22050, 22050)
    dev = Device(chunk=32)
    pool = StreamPool(dev.launch, 80, UP, 32, "cpu", resample=resample, append=dev.append, reach=REACH)
    h = pool.open(sample_rate=8000, encoding="ulaw")
    fed = 0
    for m in (5, 40, 3, 60, 9):
        fed = _feed(pool, dev, h, m, fed)
        pool.step()
    pool.close(h)
    while len(pool):
        pool.step()
    rs = Resampler(22050, 8000)
    j = 0
    for rec in seen:
        assert rec[6] == j and rec[7] >= j and rec[8].fs_out == 8000 and rec[9] == L.RESAMPLE_ULAW
        j = rec[7]
    assert j == rs.n_out(fed * UP)
