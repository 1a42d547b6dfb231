"""GPU: every public entry point on side and concurrent CUDA streams.

The contract (docstrings of FastSpeech2.forward, Generator.forward / stream / stream_pool and Resampler): a call enqueues all of its
device work on the stream current at that call; the tensors a caller passes in and gets back follow torch's usual rule; state the
library keeps between calls (packed weights, position tables, resampler taps, workspaces, stream() iterator and pool state) is ready
on whatever stream the next call uses and is not freed or reused while another stream's queued work reads it.

A stream is held busy by torch.cuda._sleep (hold), so that work queued on it behind the hold runs late.  Inputs are NaN (0 for
integers) until the side stream, after a hold, copies the real values in: a launch that goes to any other stream reads NaN.  The bar
is bit-for-bit equality with the same call on the default stream.  Every hold is at most 50 ms and nothing is repeated."""
import ctypes

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, dropin, ops, packing, synth
from fastspeech2_b200.model import FastSpeech2
from fastspeech2_b200.resample import Resampler
from tests.test_gpu_stream_vocoder import _generator

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")
HOLD_MS = 20
_CYCLES_PER_MS = []


def _cycles_per_ms():
    """torch.cuda._sleep cycles per millisecond, timed once with events."""
    if not _CYCLES_PER_MS:
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 10_000_000
        a.record()
        torch.cuda._sleep(n)
        b.record()
        b.synchronize()
        _CYCLES_PER_MS.append(n / max(a.elapsed_time(b), 1e-3))
    return _CYCLES_PER_MS[0]


def hold(s, ms=HOLD_MS):
    """Keeps stream s busy for about `ms` milliseconds: its work queued after this runs after that."""
    assert 0 < ms <= 50
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(ms * _cycles_per_ms()))


@pytest.fixture(autouse=True)
def _synchronized():
    torch.cuda.synchronize()
    yield
    torch.cuda.synchronize()


def staged(s, xs):
    """Device buffers that hold NaN (0 for integer tensors) until stream s, after a hold, copies xs into them.  The values reach the
    device first: a copy from pageable host memory would synchronise s, and so end the hold, before the call under test."""
    srcs = [x.to(DEV) if isinstance(x, torch.Tensor) else x for x in xs]
    bufs = [torch.full_like(x, NAN if x.is_floating_point() else 0) if isinstance(x, torch.Tensor) else x for x in srcs]
    torch.cuda.synchronize()
    hold(s)
    with torch.cuda.stream(s):
        for b, x in zip(bufs, srcs):
            if isinstance(x, torch.Tensor):
                b.copy_(x)
    return bufs


def same(a, b, where="out"):
    """a and b bit for bit (NaN where the other is NaN), through dicts, tuples, lists and numpy arrays."""
    if isinstance(a, dict):
        assert isinstance(b, dict) and sorted(a, key=str) == sorted(b, key=str), where
        for k in a:
            same(a[k], b[k], f"{where}[{k!r}]")
    elif isinstance(a, (tuple, list)):
        assert isinstance(b, (tuple, list)) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            same(x, y, f"{where}[{i}]")
    elif isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape, where
        torch.testing.assert_close(b.cpu(), a.cpu(), rtol=0, atol=0, equal_nan=True, msg=where)
    elif isinstance(a, np.ndarray):
        assert np.array_equal(a, b), where
    else:
        assert a == b, where


def side_equals_default(run, inputs, s):
    """run(*inputs) on the default stream, then on stream s with its inputs behind a hold: the same bits.  run must not synchronise
    the host with s before its launches (no copy from pageable host memory, no read of a device value)."""
    want = run(*[x.to(DEV) if isinstance(x, torch.Tensor) else x for x in inputs])
    torch.cuda.synchronize()
    bufs = staged(s, inputs)
    with torch.cuda.stream(s):
        got = run(*bufs)
    torch.cuda.synchronize()
    same(want, got)


@pytest.fixture(scope="module")
def side():
    return torch.cuda.Stream()


def _rnd(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


@pytest.fixture(scope="module")
def fs2(lj_configs):
    pc, mc = lj_configs
    m = FastSpeech2(pc, mc)
    m.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=31))
    return m.to(DEV).eval()


@pytest.fixture(scope="module")
def gens():
    return {"v1": _generator(configs.HIFIGAN_CONFIG, seed=3), "v2": _generator(configs.HIFIGAN_V2_CONFIG, seed=4),
            "v1b": _generator(configs.HIFIGAN_CONFIG, seed=5), "wide": _generator(configs.HIFIGAN_CONFIG, seed=3, wide_pairs=True)}


# ---------------------------------------------------------------------------------------------------- 1. side stream == default
def _op_cases():
    """name -> (run, inputs): the operator's constants on the device, its inputs on the host."""
    D = lambda t: t.to(DEV)
    x64, w = _rnd(2, 70, 64, seed=1), _rnd(3, 64, 96, seed=2, scale=0.1)
    bias, lens = D(_rnd(96, seed=3, scale=0.1)), torch.tensor([70, 41], dtype=torch.int32)
    xs, ws = _rnd(2, 60, 256, seed=4), _rnd(1, 256, 64, seed=5, scale=1 / 16)
    w_tc, w_f8 = D(packing.pack_conv_tc(w)), D(packing.pack_conv_tc(w, f8=True))
    w_seg = D(packing.pack_conv_tc_segments(ws))
    w, ws = D(w), D(ws)
    conv = lambda x, l, **kw: ops.conv1d(x, w, bias, pad_left=1, row_lens=l, **kw)
    kernels, dils = (3, 7, 11), ((1, 3, 5),) * 3
    rw = [[packing.conv_w(_rnd(32, 32, k, seed=10 + 3 * j + d, scale=0.6 * (32 * k) ** -0.5)) for d in range(3)] for j, k in enumerate(kernels)]
    rb = [[_rnd(32, seed=40 + 3 * j + d, scale=0.05).to(DEV) for d in range(3)] for j in range(3)]
    rt = [[packing.pack_conv_tc(w_, f8=True).to(DEV) for w_ in row] for row in rw]
    qkv, kl = _rnd(2, 150, 3 * 256, seed=6), torch.tensor([150, 97], dtype=torch.int32)
    g, b = D(1 + _rnd(256, seed=7, scale=0.1)), D(_rnd(256, seed=8, scale=0.1))
    table, pos = D(_rnd(50, 256, seed=9)), _rnd(200, 256, seed=11)
    ids = torch.randint(1, 50, (2, 30), generator=torch.Generator().manual_seed(12))
    spk_t, spk = D(_rnd(4, 256, seed=13)), torch.tensor([3, 1])
    hw, hb = D(_rnd(256, seed=14, scale=0.05)), D(_rnd(1, seed=15))
    bins, emb = D(torch.linspace(-1, 1, 255)), D(_rnd(256, 256, seed=16))
    cum = torch.tensor([[3, 5, 9], [2, 2, 7]], dtype=torch.int32)
    pw, pb = D(_rnd(7, 32, seed=17, scale=0.1)), D(_rnd(1, seed=18, scale=0.1))
    wav = _rnd(2, 5000, seed=19, scale=0.5)
    return {
        "conv1d_simt": (lambda x, l: conv(x, l, backend=1), (x64, lens)),
        "conv1d_tc": (lambda x, l: conv(x, l, w_tc=w_tc, backend=2), (x64, lens)),
        "conv1d_f8": (lambda x, l: conv(x, l, w_tc=w_f8, backend=2, tc_variant=1), (x64, lens)),
        "conv1d_segmented": (lambda x, l: ops.conv1d(x, ws, None, row_lens=l, w_tc=w_seg, backend=2, tc_variant=2 | 4),
                             (xs, torch.tensor([60, 33], dtype=torch.int32))),
        "resstack": (lambda x: ops.resstack(x, kernels, dils, rt, rb, rt, rb), (_rnd(2, 500, 32, seed=20),)),
        "attention_0": (lambda q, k: ops.attention(q, 2, k, backend=0), (qkv, kl)),
        "attention_2": (lambda q, k: ops.attention(q, 2, k, backend=2), (qkv, kl)),
        "layernorm": (lambda x, l: ops.layernorm(x, g, b, l), (_rnd(2, 90, 256, seed=21), torch.tensor([90, 50], dtype=torch.int32))),
        "embed_add_positions_speaker": (lambda i, p, x, s_: (ops.embed_positions(i, table, p),
                                                           ops.add_positions_(x.clone(), p), ops.add_speaker_(x.clone(), spk_t, s_)),
                                        (ids, pos, _rnd(2, 30, 256, seed=22), spk)),
        "variance_head": (lambda h, l, x: (ops.variance_head(h, hw, hb, l, 1.3, bins=bins, emb=emb, x=x), x),
                          (_rnd(2, 30, 256, seed=23), torch.tensor([30, 17], dtype=torch.int32), _rnd(2, 30, 256, seed=24))),
        "durations_length_regulate": (lambda s_, x, c: (ops.durations(s_, d_control=1.5), ops.length_regulate(x, c, 10)),
                                      (_rnd(2, 30, seed=25), _rnd(2, 3, 8, seed=26), cum)),
        "transpose": (ops.transpose_bct_to_btc, (_rnd(2, 80, 33, seed=27),)),
        "conv_post": (lambda x, l: ops.conv_post(x, pw, pb, 0.01, l, 4), (_rnd(2, 400, 32, seed=28), torch.tensor([100, 61], dtype=torch.int32))),
        "wav_to_int16": (lambda w_, l: ops.wav_to_int16(w_, l), (wav, torch.tensor([5000, 1234]))),
    }


OP_CASES = [
    "conv1d_simt", "conv1d_tc", "conv1d_f8", "conv1d_segmented", "resstack", "attention_0", "attention_2", "layernorm",
    "embed_add_positions_speaker", "variance_head", "durations_length_regulate", "transpose", "conv_post", "wav_to_int16"]


@pytest.mark.parametrize("name", OP_CASES)
def test_ops_on_side_stream(name, side):
    run, inputs = _op_cases()[name]
    side_equals_default(run, inputs, side)


def _teacher(batch, seed):
    """Teacher-forcing targets for a make_batch batch: (mel_lens, max_mel_len, p_targets, e_targets, d_targets)."""
    _, texts, lens, Lm = batch
    g = torch.Generator().manual_seed(seed)
    d = torch.randint(0, 6, (len(lens), Lm), generator=g).float() * (torch.arange(Lm)[None, :] < lens[:, None])
    mel_lens = d.sum(1).long()
    return mel_lens, int(mel_lens.max()), torch.randn(len(lens), Lm, generator=g), torch.randn(len(lens), Lm, generator=g), d


FS2_CASES = ["padded", "ragged", "teacher_forced", "max_mel_len", "ragged_max_mel_len"]


@pytest.mark.parametrize("case", FS2_CASES)
def test_fastspeech2_on_side_stream(case, fs2, side):
    batch = synth.make_batch(4, 40, seed=32, min_len=9)
    spk, texts, lens, Lm = batch
    ragged = case.startswith("ragged")
    if case == "teacher_forced":
        mel_lens, T, p_t, e_t, d_t = _teacher(batch, seed=33)
        run = lambda s_, t, l, ml, p, e, d: fs2(s_, t, l, Lm, None, ml, T, p, e, d)
        side_equals_default(run, (spk, texts, lens, mel_lens, p_t, e_t, d_t), side)
        return
    T = None
    if case.endswith("max_mel_len"):
        T = int(fs2(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm, ragged=ragged)[9].max()) + 3
    side_equals_default(lambda s_, t, l: fs2(s_, t, l, Lm, max_mel_len=T, ragged=ragged), (spk, texts, lens), side)


@pytest.mark.parametrize("case", ["v1", "v2", "v1_ragged", "v2_ragged", "wide"])
def test_generator_on_side_stream(case, gens, side):
    gen = gens[case.split("_")[0]]
    mel = synth.make_mel(3, 45, seed=34)
    if case.endswith("ragged"):
        side_equals_default(lambda x, l: gen(x, l), (mel, torch.tensor([45, 20, 1])), side)
    else:
        side_equals_default(gen, (mel,), side)


@pytest.mark.parametrize("fmt", [{}, {"sample_rate": 16000}, {"pcm16": True}, {"sample_rate": 8000, "pcm16": True}])
def test_generator_stream_on_side_stream(fmt, gens, side):
    gen = gens["v1"]
    run = lambda x, l: list(gen.stream(x, mel_lens=l, chunk_frames=16, **fmt))
    side_equals_default(run, (synth.make_mel(2, 50, seed=35), torch.tensor([50, 29])), side)


def _drive_pool(pool, mels, formats=None, opened=(), generators=None):
    """Adds mels[k] (format formats[k], generator generators[k]) before step k, opens streams fed block by block (mel, blocks)
    from step 0, closing each after its last block, and steps to the end: every stream's list of (first_sample, chunk)."""
    handles, parts, blocks = {}, {}, {}
    for k, (mel, sizes) in enumerate(opened):
        handles[pool.open()] = ("open", k)
        blocks[k] = list(sizes)
    step, fed = 0, {k: 0 for k in blocks}
    while step < len(mels) or len(pool):
        if step < len(mels):
            kw = dict(formats[step]) if formats else {}
            if generators:
                kw["generator"] = generators[step]
            handles[pool.add(mels[step], **kw)] = step
        for h, key in list(handles.items()):
            if isinstance(key, tuple) and blocks[key[1]]:
                m = blocks[key[1]].pop(0)
                mel = opened[key[1]][0]
                pool.feed(h, mel[:, fed[key[1]]:fed[key[1]] + m])
                fed[key[1]] += m
                if not blocks[key[1]]:
                    pool.close(h)
        for h, start, y in pool.step():
            parts.setdefault(handles[h], []).append((start, y))
        step += 1
    return parts


def test_stream_pool_on_side_stream(gens, side):
    """add() (a contiguous [80, n] mel: converted), open / feed / close, mixed rates and encodings, and a second generator."""
    v1, v1b = gens["v1"], gens["v1b"]
    formats = [{}, {"sample_rate": 16000}, {"encoding": "ulaw", "sample_rate": 8000}, {"encoding": "pcm16"}]
    mels = [synth.make_mel(1, n, seed=36 + i)[0] for i, n in enumerate((70, 33, 52, 20))]
    fed = synth.make_mel(1, 60, seed=40)[0]

    def run(a, b, c, d, f):
        pool = v1.stream_pool(chunk_frames=16, generators=(v1b,))
        return _drive_pool(pool, [a, b, c, d], formats, opened=[(f, [25, 1, 34])], generators=[0, 1, 0, 1])
    side_equals_default(run, (*mels, fed), side)


@pytest.mark.parametrize("call", ["call", "window", "streams", "mixed"])
def test_resampler_on_side_stream(call, side):
    rs = Resampler(22050, 16000)
    x = _rnd(2, 3000, seed=41, scale=0.3)
    if call == "call":
        side_equals_default(lambda w, l: (rs(w, l), rs(w, l, pcm16=True)), (x, torch.tensor([3000, 1700])), side)
    elif call == "window":
        side_equals_default(lambda w: rs.window(w[:, :1000], w[:, 1000:2000], 1000, 3000, 100, 900), (x,), side)
    elif call == "streams":
        def run(w):
            recs = [(w[b].data_ptr(), w[b, 1000:].data_ptr(), 0, 1000, 3000, 3000, 0, 1500) for b in range(2)]
            return rs.streams(recs, 1500, DEV)
        side_equals_default(run, (x,), side)
    else:
        other = Resampler(22050, 8000)

        def run(w):
            recs = [(w[0].data_ptr(), w[0, 1000:].data_ptr(), 0, 1000, 3000, 3000, 0, 1500, rs, L.RESAMPLE_F32),
                    (w[1].data_ptr(), w[1, 1000:].data_ptr(), 0, 1000, 3000, 3000, 0, 800, other, L.RESAMPLE_ULAW)]
            y, views = Resampler.mixed(recs, 1500, DEV)
            return [v.clone() for v in views]
        side_equals_default(run, (x,), side)


def test_vocoder_infer_on_side_stream(lj_configs, gens, side):
    """Device lengths, not ragged: nothing reads a device value before the vocoder's launches."""
    pc, mc = lj_configs
    run = lambda x, l: dropin.vocoder_infer(x, gens["v1"], mc, pc, lengths=l)
    side_equals_default(run, (synth.make_mel(2, 30, seed=42), torch.tensor([30 * 256, 11 * 256])), side)


# ---------------------------------------------------------------------------------------------------- 2. state crossing streams
@pytest.fixture(scope="module")
def s2():
    return torch.cuda.Stream()


def test_first_call_packs_on_one_stream_second_call_on_another(lj_configs, side, s2):
    """Packing on s1 behind a hold, then a call on s2 straight away.  packing.split_fp16 reads each layer's max to the host, which
    absorbs the hold, so only the device work after the last such read is still queued on s1: this guards the packed weights'
    event rather than catching a fault of the code it was written against."""
    pc, mc = lj_configs
    sd, hsd = synth.fastspeech2_state_dict(pc, mc, seed=43), synth.hifigan_state_dict(configs.HIFIGAN_CONFIG, seed=44)

    def fresh():
        m = FastSpeech2(pc, mc)
        m.load_state_dict(sd)
        return m.to(DEV).eval(), _generator(configs.HIFIGAN_CONFIG, sd=hsd)
    spk, texts, lens, Lm = [x.to(DEV) if isinstance(x, torch.Tensor) else x for x in synth.make_batch(2, 30, seed=45)]
    mel = synth.make_mel(2, 40, seed=46).to(DEV)
    ref_m, ref_g = fresh()
    want_m, want_g = ref_m(spk, texts, lens, Lm, max_mel_len=90), ref_g(mel)
    torch.cuda.synchronize()
    m, g = fresh()
    hold(side)
    with torch.cuda.stream(side):
        got1 = (m(spk, texts, lens, Lm, max_mel_len=90), g(mel))
    with torch.cuda.stream(s2):
        got2 = (m(spk, texts, lens, Lm, max_mel_len=90), g(mel))
    torch.cuda.synchronize()
    same((want_m, want_g), got1)
    same((want_m, want_g), got2)


def test_resampler_taps_uploaded_on_one_stream_read_on_another(side, s2):
    """The taps' upload from pageable host memory synchronises s1, which ends the hold, so this guards the taps' event rather than
    catching a fault of the code it was written against."""
    x = _rnd(2, 2000, seed=47, scale=0.3).to(DEV)
    want = Resampler(22050, 24000)(x)
    torch.cuda.synchronize()
    rs = Resampler(22050, 24000)
    hold(side)
    with torch.cuda.stream(side):
        got1 = rs(x)                                  # uploads the taps on s1, behind the hold
    with torch.cuda.stream(s2):
        got2 = rs(x)
    torch.cuda.synchronize()
    same(want, got1)
    same(want, got2)


@pytest.mark.parametrize("fmt", [{}, {"sample_rate": 16000}])
def test_stream_made_on_one_stream_consumed_on_another(fmt, gens, side, s2):
    """A [B, 80, T] contiguous mel, so that stream() transposes it (on s1, behind a hold), and every chunk consumed on s2."""
    gen = gens["v1"]
    mel = synth.make_mel(2, 70, seed=48 + len(fmt))         # another mel per case: a stale transpose of the last one differs
    want = list(gen.stream(mel.to(DEV), chunk_frames=16, **fmt))
    torch.cuda.synchronize()
    (buf,) = staged(side, (mel,))
    with torch.cuda.stream(side):
        it = gen.stream(buf, chunk_frames=16, **fmt)
    with torch.cuda.stream(s2):
        got = list(it)
    torch.cuda.synchronize()
    same(want, got)


def test_pool_driven_from_two_streams(gens, side, s2):
    """add / feed on s1 behind holds, and steps alternating between s1 and s2 with a hold on s1 before each."""
    gen = gens["v1"]
    mels = [synth.make_mel(1, n, seed=50 + i)[0].to(DEV) for i, n in enumerate((60, 35, 47))]
    fed = synth.make_mel(1, 52, seed=53)[0].to(DEV)
    formats = [{}, {"sample_rate": 16000}, {"encoding": "pcm16"}]
    want = _drive_pool(gen.stream_pool(chunk_frames=16), mels, formats, opened=[(fed, [20, 32])])
    torch.cuda.synchronize()

    pool = gen.stream_pool(chunk_frames=16)
    handles, parts = {}, {}
    hold(side)
    with torch.cuda.stream(side):
        h_open = pool.open()
        handles[h_open] = ("open", 0)
    blocks, k, step = [20, 32], 0, 0
    while step < len(mels) or len(pool):
        hold(side)
        with torch.cuda.stream(side):
            if step < len(mels):
                handles[pool.add(mels[step], **formats[step])] = step     # contiguous [80, n]: converted on s1
            if blocks:
                m = blocks.pop(0)
                pool.feed(h_open, fed[:, k:k + m].half())                  # fp16: converted on s1
                k += m
                if not blocks:
                    pool.close(h_open)
        with torch.cuda.stream(side if step % 2 == 0 else s2):
            for h, start, y in pool.step():
                parts.setdefault(handles[h], []).append((start, y))
        step += 1
    torch.cuda.synchronize()
    # the fp16 feed rounds the fed stream's mel: compare it against the default-stream pool fed the same fp16 blocks
    want_fed = _drive_pool(gen.stream_pool(chunk_frames=16), [], opened=[(fed.half().float(), [20, 32])])
    torch.cuda.synchronize()
    same({k_: v for k_, v in want.items() if k_ != ("open", 0)}, {k_: v for k_, v in parts.items() if k_ != ("open", 0)})
    same(want_fed[("open", 0)], parts[("open", 0)])


def test_long_position_table_built_on_one_stream(lj_configs, side, s2):
    """T > max_seq_len: the decoder's position table is built by the first such call (on s1, behind a hold) and read on s2.  The
    table's upload from pageable host memory synchronises s1 as the resampler's taps do; the rest of both calls overlaps."""
    pc, mc = lj_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=54)
    spk, texts, lens, Lm = [x.to(DEV) if isinstance(x, torch.Tensor) else x for x in synth.make_batch(2, 20, seed=55)]
    T = int(mc["max_seq_len"]) + 100

    def fresh():
        m = FastSpeech2(pc, mc)
        m.load_state_dict(sd)
        m = m.to(DEV).eval()
        m(spk, texts, lens, Lm, max_mel_len=50)           # packs on the default stream
        torch.cuda.synchronize()
        return m
    want = fresh()(spk, texts, lens, Lm, max_mel_len=T)
    m = fresh()
    hold(side)
    with torch.cuda.stream(side):
        got1 = m(spk, texts, lens, Lm, max_mel_len=T)
    with torch.cuda.stream(s2):
        got2 = m(spk, texts, lens, Lm, max_mel_len=T)
    torch.cuda.synchronize()
    same(want, got1)
    same(want, got2)


# ---------------------------------------------------------------------------------------------------- 3. workspaces not reused early
PATTERN = 0x5A


def _probes(nbytes, n=8):
    """n tensors of nbytes, allocated on the current stream and filled with PATTERN."""
    return [torch.full((int(nbytes),), PATTERN, dtype=torch.uint8, device=DEV) for _ in range(n)]


def _intact(probes):
    for i, p in enumerate(probes):
        assert bool((p == PATTERN).all()), f"probe {i} was written by a call on another stream"


def test_generator_workspace_not_reused_while_another_stream_uses_it(side):
    """Default stream: a call, sync.  s1: hold, a same-size call.  Default: a larger call, then probes of the first workspace's
    size.  After a sync the probes hold their pattern and s1's output equals the default stream's.  The same sequence runs once
    first, unheld, on a twin generator, so that every block the held run allocates is already cached: a cudaMalloc inside the held
    run could wait for the device and end the overlap, and the probes then take each cached block of their size."""
    small, large = synth.make_mel(2, 40, seed=56).to(DEV), synth.make_mel(6, 40, seed=57).to(DEV)
    twins = [_generator(configs.HIFIGAN_V2_CONFIG, seed=4) for _ in range(2)]
    m = twins[0]._pack()[0]
    twins[1]._pack()
    nbytes = L.lib().fs2_vocoder_workspace_bytes(ctypes.byref(m), 2, 40) + 1024

    def sequence(gen, held):
        want = gen(small)
        torch.cuda.synchronize()
        if held:
            hold(side)
        with torch.cuda.stream(side):
            got = gen(small)
        gen(large)
        probes = _probes(nbytes)
        torch.cuda.synchronize()
        return want, got, probes
    sequence(twins.pop(0), held=False)
    want, got, probes = sequence(twins.pop(0), held=True)
    _intact(probes)
    same(want, got)


def test_fastspeech2_workspace_not_reused_while_another_stream_uses_it(lj_configs, side):
    pc, mc = lj_configs
    fs2 = FastSpeech2(pc, mc)
    fs2.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=31))
    fs2 = fs2.to(DEV).eval()
    small = [x.to(DEV) if isinstance(x, torch.Tensor) else x for x in synth.make_batch(2, 40, seed=58)]
    large = [x.to(DEV) if isinstance(x, torch.Tensor) else x for x in synth.make_batch(8, 40, seed=59)]
    T = 200
    want = fs2(*small, max_mel_len=T)
    torch.cuda.synchronize()
    m = fs2._packed[0]
    lib = L.lib()
    old = max(lib.fs2_encode_workspace_bytes(ctypes.byref(m), 2, small[3]), lib.fs2_decode_workspace_bytes(ctypes.byref(m), 2, T))
    hold(side)
    with torch.cuda.stream(side):
        got = fs2(*small, max_mel_len=T)
    fs2(*large, max_mel_len=T)
    probes = _probes(int(old * 1.25) + 1024)
    torch.cuda.synchronize()
    _intact(probes)
    same(want, got)


def test_pool_workspace_not_reused_while_another_stream_uses_it(gens, side):
    """A pool stepped on the default stream, then on s1 behind a hold, then on the default stream with more live streams."""
    gen = gens["v1"]
    mels = [synth.make_mel(1, 48, seed=60 + i)[0].T.contiguous().to(DEV).T for i in range(6)]   # channels-last views: no copy
    want = _drive_pool(gen.stream_pool(chunk_frames=16), mels[:2])
    torch.cuda.synchronize()

    pool = gen.stream_pool(chunk_frames=16)
    handles, parts = {pool.add(mels[0]): 0, pool.add(mels[1]): 1}, {}
    for h, start, y in pool.step():                      # default stream: 2 live
        parts.setdefault(handles[h], []).append((start, y))
    torch.cuda.synchronize()
    hold(side)
    with torch.cuda.stream(side):                        # s1: 2 live, behind the hold
        for h, start, y in pool.step():
            parts.setdefault(handles[h], []).append((start, y))
    for k in range(2, 6):                                # default: 6 live
        handles[pool.add(mels[k])] = k
    for h, start, y in pool.step():
        parts.setdefault(handles[h], []).append((start, y))
    m = gen._packed[0]
    probes = _probes(L.lib().fs2_vocoder_streams_workspace_bytes(ctypes.byref(m), 2, 16))
    while len(pool):
        for h, start, y in pool.step():
            parts.setdefault(handles[h], []).append((start, y))
    torch.cuda.synchronize()
    _intact(probes)
    alone = {k: _drive_pool(gen.stream_pool(chunk_frames=16), [mels[k]])[0] for k in range(2, 6)}
    torch.cuda.synchronize()
    same(want[0], parts[0])
    same(want[1], parts[1])
    for k in range(2, 6):
        same([y for _, y in alone[k]], [y for _, y in parts[k]])


# ---------------------------------------------------------------------------------------------------- 4. two streams at once
def test_full_size_calls_on_two_streams_at_once(fs2, gens, side, s2):
    """s1 and s2 held for the same time, then a full-size (B = 16 x 1012 frames) Generator call and a FastSpeech2 call on each: both
    equal their serial outputs.  How much the two streams overlap is up to the GPU's scheduler, so this test shows that concurrent
    calls share no state when they do overlap; it is not a deterministic detector of shared state."""
    gen = gens["v1"]
    mels = [synth.make_mel(16, 1012, seed=70 + i).to(DEV) for i in range(2)]
    batches = [[x.to(DEV) if isinstance(x, torch.Tensor) else x for x in synth.make_batch(16, 128, seed=72 + i)] for i in range(2)]
    want = [(gen(mels[i]), fs2(*batches[i])) for i in range(2)]
    torch.cuda.synchronize()
    Ts = [int(w[1][9].max()) for w in want]
    hold(side, 40)
    hold(s2, 40)
    got = []
    for i, s in enumerate((side, s2)):
        with torch.cuda.stream(s):
            got.append((gen(mels[i]), fs2(*batches[i], max_mel_len=Ts[i])))
    torch.cuda.synchronize()
    for i in range(2):
        same(want[i], got[i], f"stream {i + 1}")
