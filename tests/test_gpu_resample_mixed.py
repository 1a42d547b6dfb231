"""GPU: streams at their own output rates and encodings in one resampling launch (fs2_resample_streams_mixed, StreamPool.add(...,
sample_rate, encoding)), bit for bit against the offline resampler of each stream alone and the numpy G.711 oracle, whatever shares the
pool, in at most one conversion launch per tick."""
import ctypes

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, ops, synth
from fastspeech2_b200.resample import ENCODINGS, Resampler
from tests.test_gpu_stream_vocoder import _generator
from tests.test_resample_mixed_cpu import ALL_INT16, g711_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
FS_IN = 22050
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
FORMATS = ((8000, "ulaw"), (8000, "alaw"), (16000, "pcm16"), (22050, "pcm16"), (22050, "f32"), (24000, "f32"), (44100, "pcm16"),
           (48000, "f32"))
LENS = (70, 5, 37, 90, 1, 44, 61, 23)
JOIN = (0, 2, 2, 1, 3, 0, 4, 1)


def _offline(gen, mel, rate, encoding):
    """What one stream's concatenated chunks must equal: the offline resampler of the offline forward, G.711 from its PCM16."""
    pcm = encoding != "f32"
    y = Resampler(FS_IN, rate)(gen(mel[None]), pcm16=pcm)
    if encoding in ("ulaw", "alaw"):
        y = torch.from_numpy(g711_ref(y.cpu().numpy().astype(np.int64), ENCODINGS[encoding])).to(DEV)
    return y


def _run(pool, mels, formats, join, cancel_at=None, cancel=None):
    handles, parts, first = {}, {}, {}
    step = 0
    while step <= max(join) or len(pool):
        for k, j in enumerate(join):
            if j == step:
                handles[pool.add(mels[k], sample_rate=formats[k][0], encoding=formats[k][1])] = k
        if step == cancel_at:
            pool.cancel(next(h for h, k in handles.items() if k == cancel))
        for h, start, y in pool.step():
            k = handles[h]
            assert start == first.get(k, 0) and y.dim() == 3 and y.shape[:2] == (1, 1)
            assert y.dtype == {"f32": torch.float32, "pcm16": torch.int16}.get(formats[k][1], torch.uint8)
            first[k] = start + y.shape[2]
            parts.setdefault(k, []).append(y)
        step += 1
    return {k: (torch.cat(v, dim=2), len(v)) for k, v in parts.items()}


@pytest.mark.parametrize("cfg", list(CFGS))
def test_mixed_pool_equals_offline(cfg):
    gen = _generator(CFGS[cfg])
    mels = [synth.make_mel(1, n, seed=200 + i)[0].to(DEV) for i, n in enumerate(LENS)]
    chunk = 16
    got = _run(gen.stream_pool(chunk_frames=chunk), mels, FORMATS, JOIN, cancel_at=3, cancel=0)
    for k, mel in enumerate(mels):
        if k == 0:
            assert got[k][1] == 3                                  # cancelled after three chunks
            continue
        y, n_chunks = got[k]
        assert n_chunks == -(-LENS[k] // chunk)
        assert torch.equal(y, _offline(gen, mel, *FORMATS[k])), (k, FORMATS[k])


def test_batch_invariance():
    """One 16 kHz PCM16 stream and one 8 kHz mu-law stream give the same bytes alone, in a pool of their own format, and in a
    permuted mix joining at other ticks."""
    gen = _generator(CFGS["v1"])
    mels = [synth.make_mel(1, n, seed=300 + i)[0].to(DEV) for i, n in enumerate(LENS)]
    chunk = 8
    mix = _run(gen.stream_pool(chunk_frames=chunk), mels, FORMATS, JOIN)
    perm = [5, 2, 7, 0, 3, 6, 1, 4]
    mixed2 = _run(gen.stream_pool(chunk_frames=chunk), [mels[p] for p in perm], [FORMATS[p] for p in perm], (1, 0, 0, 3, 2, 1, 0, 2))
    for k in (2, 0):
        rate, enc = FORMATS[k]
        alone = _run(gen.stream_pool(chunk_frames=chunk), [mels[k]], [FORMATS[k]], (0,))
        same = _run(gen.stream_pool(chunk_frames=chunk, sample_rate=rate, pcm16=enc == "pcm16"), [mels[k], mels[3], mels[6]],
                    [FORMATS[k]] * 3, (0, 0, 1))
        want = mix[k][0]
        assert torch.equal(alone[0][0], want) and torch.equal(same[0][0], want) and torch.equal(mixed2[perm.index(k)][0], want), k


def _mixed_call(records, filters, n_out_bytes, max_out, n_filters=None, sentinel=0xAB):
    """A raw fs2_resample_streams_mixed call: records are ResampleMixedStream field tuples; returns the output buffer."""
    B = len(records)
    host = (L.ResampleMixedStream * B)(*[L.ResampleMixedStream(*r) for r in records])
    table = torch.frombuffer(bytearray(bytes(host)), dtype=torch.uint8).to(DEV)
    y = torch.full((n_out_bytes,), sentinel, dtype=torch.uint8, device=DEV)
    a = L.ResampleMixedArgs(B=B, n_filters=len(filters) if n_filters is None else n_filters, table=table.data_ptr(), max_out=max_out,
                            y=y.data_ptr(), scale=32768.0)
    for i, f in enumerate(filters):
        a.filters[i] = L.ResampleFilter(**f._filter(DEV))
    L.check(L.lib().fs2_resample_streams_mixed(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "mixed")
    torch.cuda.synchronize()
    return y


def test_kernel_rows_equal_the_window_call():
    """Rows of random filters (the identity among them), encodings and output ranges in one call: each equals fs2_resample_window of
    its row alone (the identity: the input itself, or its wav_to_int16), G.711 rows the oracle of that PCM16."""
    rng = np.random.default_rng(7)
    rates = (8000, 16000, 22050, 24000, 44100, 48000, 11025, 32000)
    filters = [Resampler(FS_IN, r) for r in rates]
    recs, want, xs = [], [], []
    off, max_out = 0, 0
    for b in range(24):
        f = int(rng.integers(0, len(filters)))
        enc = int(rng.integers(0, 4))
        rs = filters[f]
        N = int(rng.integers(1, 30000))
        x = (torch.from_numpy(rng.standard_normal(N).astype(np.float32)) * 0.6).to(DEV)
        xs.append(x)
        n_out = rs.n_out(N)
        j0 = int(rng.integers(0, n_out))
        j1 = int(rng.integers(j0 + 1, n_out + 1))
        if rs.identity:
            ref = x[j0:j1]
            ref = ops.wav_to_int16(ref[None].contiguous())[0] if enc else ref
        else:
            ref = rs.window(None, x[None], 0, N, j0, j1, pcm16=bool(enc))[0]
        if enc >= L.RESAMPLE_ULAW:
            ref = torch.from_numpy(g711_ref(ref.cpu().numpy().astype(np.int64), enc)).to(DEV)
        want.append(ref)
        recs.append((0, x.data_ptr(), 0, 0, N, N, j0, j1, f, enc, off))
        off += -(-(j1 - j0) * ref.element_size() // 16) * 16
        max_out = max(max_out, j1 - j0)
    y = _mixed_call(recs, filters, off, max_out)
    for b, r in enumerate(recs):
        got = y[r[10]:r[10] + want[b].numel() * want[b].element_size()].view(want[b].dtype)
        assert torch.equal(got, want[b]), (b, rates[r[8]], r[9])


def test_identity_call_equals_the_g711_oracle():
    """x = s / 32768 over every int16 s, through the identity filter: PCM16 gives s back, mu-law and A-law the oracle's codes."""
    s = torch.from_numpy(ALL_INT16.astype(np.int16))
    x = (s.float() / 32768.0).to(DEV)
    ident = Resampler(FS_IN, FS_IN)
    n = x.numel()
    recs = [(0, x.data_ptr(), 0, 0, n, n, 0, n, 0, enc, o) for enc, o in
            ((L.RESAMPLE_PCM16, 0), (L.RESAMPLE_ULAW, 2 * n), (L.RESAMPLE_ALAW, 3 * n), (L.RESAMPLE_F32, 4 * n))]
    y = _mixed_call(recs, [ident], 8 * n, n)
    assert torch.equal(y[:2 * n].view(torch.int16).cpu(), s)
    assert np.array_equal(y[2 * n:3 * n].cpu().numpy(), g711_ref(ALL_INT16, L.RESAMPLE_ULAW))
    assert np.array_equal(y[3 * n:4 * n].cpu().numpy(), g711_ref(ALL_INT16, L.RESAMPLE_ALAW))
    assert torch.equal(y[4 * n:].view(torch.float32), x)


def test_records_outside_the_table_write_nothing():
    x = torch.randn(4000, device=DEV)
    rs = Resampler(FS_IN, 16000)
    good = (0, x.data_ptr(), 0, 0, 4000, 4000, 0, 100)
    recs = [good + (2, 0, 0),          # filter index past n_filters = 2 (the table has a third entry, not passed)
            good + (-1, 0, 512),       # negative filter index
            good + (0, 4, 1024),       # unknown encoding
            good + (0, -1, 1536),
            good + (0, 0, 2056),       # offset not a multiple of 16
            good + (0, 0, -16),        # negative offset
            good + (1, 1, 2560)]       # the one valid record: identity, PCM16
    y = _mixed_call(recs, [rs, Resampler(FS_IN, FS_IN), Resampler(FS_IN, 8000)], 4096, 100, n_filters=2)
    assert (y[:2560] == 0xAB).all() and (y[2760:] == 0xAB).all()
    assert torch.equal(y[2560:2760].view(torch.int16), ops.wav_to_int16(x[None, :100])[0])


@pytest.mark.parametrize("cfg", list(CFGS))
def test_a_mixed_tick_adds_at_most_one_launch(cfg):
    gen = _generator(CFGS[cfg])
    m, _keep, _dev, up = gen._pack()
    frames = 32
    h = L.lib()
    mels = [synth.make_mel(1, 100, seed=400 + i)[0].to(DEV) for i in range(len(FORMATS))]
    plan = len(L.vocoder_window_plan(m, 100, 0, frames)) + 1          # the vocoder's plan plus its staging launch
    native = gen.stream_pool(chunk_frames=frames)
    for mel in mels[:3]:
        native.add(mel)
    mixed = gen.stream_pool(chunk_frames=frames)
    for mel, (rate, enc) in zip(mels, FORMATS):
        mixed.add(mel, sample_rate=rate, encoding=enc)
    for pool, extra in ((native, 0), (mixed, 1)):
        pool.step()                                                    # first tick: kernel setup
        torch.cuda.synchronize()
        n0 = h.fs2_kernel_launch_count()
        pool.step()
        torch.cuda.synchronize()
        assert h.fs2_kernel_launch_count() - n0 == plan + extra, (cfg, extra)
