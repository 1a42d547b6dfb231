"""GPU: streams of several HiFi-GAN generators in one pool (Generator.stream_pool(generators=...), fs2_vocoder_forward_streams_multi),
bit for bit against each stream's own generator's forward on that stream alone.  The bar is torch.equal throughout: the plan is
generator 0's, every output row's sums keep their order, and only where a work item reads its weights from changes."""
import ctypes

import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from tests.test_gpu_resample_mixed import _offline
from tests.test_gpu_stream_pool import _streams_call
from tests.test_gpu_stream_vocoder import _generator

pytestmark = pytest.mark.gpu
DEV = "cuda"
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
POLICIES = {"default": {}, "exact": {"use_tensor_cores": False}, "per_layer": {"fused_mask": 0, "pair_mask": 0},
            "wide_pairs": {"wide_pairs": True}}
CHUNK = 32
LENS = (70, 5, 37, 90, 1, 44, 61, 23, 33)


def _mel(n, seed):
    return synth.make_mel(1, n, seed=seed)[0].to(DEV)


def _run(pool, mels, gens, join):
    """Adds stream k (mel, generator index) at tick join[k]; runs the pool to its end and returns each stream's concatenated chunks."""
    parts, handles, tick = {}, {}, 0
    while tick <= max(join) or len(pool):
        for k, t in enumerate(join):
            if t == tick:
                handles[pool.add(mels[k], generator=gens[k])] = k
        for h, first, chunk in pool.step():
            parts.setdefault(handles[h], []).append(chunk)
        tick += 1
    return {k: torch.cat(v, dim=-1) for k, v in parts.items()}


def _check_pool(gens):
    pool = gens[0].stream_pool(chunk_frames=CHUNK, generators=gens[1:])
    mels = [_mel(n, seed=40 + k) for k, n in enumerate(LENS)]
    which = [k % len(gens) for k in range(len(LENS))]
    out = _run(pool, mels, which, [0, 0, 1, 0, 2, 1, 3, 0, 2])
    for k, mel in enumerate(mels):
        assert torch.equal(out[k], gens[which[k]](mel[None])), (k, which[k])


@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_pool_of_two_synthetic_generators_equals_each_forward(cfg, policy):
    if policy == "wide_pairs" and cfg != "v1":
        pytest.skip("wide pairs are V1's 128-channel stage")
    _check_pool([_generator(CFGS[cfg], seed=s, **POLICIES[policy]) for s in (3, 11)])


def test_pool_of_the_real_checkpoints_equals_each_forward():
    from oracle import real_ckpt
    sds = [real_ckpt.load(n) for n in ("LJSpeech", "universal")]
    if any(sd is None for sd in sds):
        pytest.skip("real-checkpoint fixtures not built (oracle/_ref/)")
    gens = [_generator(configs.HIFIGAN_CONFIG, sd=sd) for sd in sds]
    _check_pool(gens + [_generator(configs.HIFIGAN_CONFIG, seed=5)])


@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_mixed_pool_of_added_and_open_streams_and_formats(cfg):
    gens = [_generator(CFGS[cfg], seed=s) for s in (3, 11, 17)]
    pool = gens[0].stream_pool(chunk_frames=CHUNK, generators=gens[1:])
    spec = [(70, 0, None, None, "add"), (45, 1, 16000, "pcm16", "open"), (90, 2, 8000, "ulaw", "add"), (33, 1, 24000, "f32", "open"),
            (61, 0, 16000, "pcm16", "open"), (12, 2, None, None, "open")]
    mels = [_mel(n, seed=60 + k) for k, (n, *_rest) in enumerate(spec)]
    handles, parts, fed = {}, {}, {}
    for k, (n, g, rate, enc, kind) in enumerate(spec):
        if kind == "add":
            handles[pool.add(mels[k], sample_rate=rate, encoding=enc, generator=g)] = k
        else:
            handles[pool.open(sample_rate=rate, encoding=enc, generator=g)] = k
            fed[k] = 0
    tick = 0
    while len(pool):
        for h, k in handles.items():
            if k in fed and fed[k] < spec[k][0]:
                m = min(7 + 3 * k, spec[k][0] - fed[k])
                pool.feed(h, mels[k][:, fed[k]:fed[k] + m])
                fed[k] += m
                if fed[k] == spec[k][0]:
                    pool.close(h)
        for h, first, chunk in pool.step():
            parts.setdefault(handles[h], []).append(chunk.reshape(-1))
        tick += 1
        assert tick < 200
    for k, (n, g, rate, enc, kind) in enumerate(spec):
        got = torch.cat(parts[k])
        if rate is None:
            assert torch.equal(got, gens[g](mels[k][None]).reshape(-1)), k
        else:
            assert torch.equal(got, _offline(gens[g], mels[k], rate, enc).reshape(-1)), k


def _multi_call(gens, rows, lens, f0s, gen_idx, frames, n_models=None):
    """One fs2_vocoder_forward_streams_multi call; the launches it made."""
    packs = [g._packed or g._pack() for g in gens]
    models = L.model_array([p[0] for p in packs])
    models_dev = torch.frombuffer(bytearray(b"".join(bytes(p[0]) for p in packs)), dtype=torch.uint8).to(DEV)
    n = len(gens) if n_models is None else n_models
    up = packs[0][3]
    B = len(rows)
    t = lambda v, dt: torch.tensor(v, dtype=dt, device=DEV)
    ptrs, lens_d, f0_d, gen_d = t([r.data_ptr() for r in rows], torch.int64), t(lens, torch.int32), t(f0s, torch.int32), t(gen_idx, torch.int32)
    need = L.lib().fs2_vocoder_streams_multi_workspace_bytes(models, n, B, frames)
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    out = torch.full((B, frames * up), float("nan"), device=DEV)
    a = L.VocoderStreamsMultiArgs(B=B, frames=frames, mel=ptrs.data_ptr(), mel_lens=lens_d.data_ptr(), f0=f0_d.data_ptr(),
                                  wav=out.data_ptr(), wav_batch_stride=frames * up, workspace=ws.data_ptr(), workspace_bytes=need, cap=0,
                                  gen=gen_d.data_ptr(), models_dev=models_dev.data_ptr())
    torch.cuda.synchronize()
    n0 = L.lib().fs2_kernel_launch_count()
    L.check(L.lib().fs2_vocoder_forward_streams_multi(models, n, ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "multi")
    launches = L.lib().fs2_kernel_launch_count() - n0
    torch.cuda.synchronize()
    return out, launches


@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_one_model_multi_call_equals_the_streams_call_and_launches_as_many_kernels(cfg):
    gens = [_generator(CFGS[cfg], seed=s) for s in (3, 11)]
    lens = [90, 40, 70, 12, 55]
    rows = [_mel(n, seed=80 + b).T.contiguous() for b, n in enumerate(lens)]
    f0s = [32, 0, 64, 0, 50]
    n0 = L.lib().fs2_kernel_launch_count()
    ref = _streams_call(gens[0], rows, lens, f0s, CHUNK)
    one_launches = L.lib().fs2_kernel_launch_count() - n0
    out, launches1 = _multi_call(gens[:1], rows, lens, f0s, [0] * len(rows), CHUNK)
    assert torch.equal(out, ref)
    two, launches2 = _multi_call(gens, rows, lens, f0s, [1, 0, 1, 1, 0], CHUNK)
    assert launches1 == launches2 == one_launches
    ref1 = _streams_call(gens[1], rows, lens, f0s, CHUNK)
    for b, g in enumerate([1, 0, 1, 1, 0]):
        assert torch.equal(two[b], (ref1 if g else ref)[b]), b


def test_out_of_range_generator_index_gives_a_zero_chunk_and_leaves_the_others():
    gens = [_generator(configs.HIFIGAN_CONFIG, seed=s) for s in (3, 11)]
    lens = [90, 40, 70, 55]
    rows = [_mel(n, seed=90 + b).T.contiguous() for b, n in enumerate(lens)]
    f0s = [0, 0, 32, 16]
    good, _ = _multi_call(gens, rows, lens, f0s, [1, 0, 1, 0], CHUNK)
    for bad in (2, -1, 1 << 30):
        out, _ = _multi_call(gens, rows, lens, f0s, [1, bad, 1, 0], CHUNK)
        assert torch.equal(out[1], torch.zeros_like(out[1])), bad
        for b in (0, 2, 3):
            assert torch.equal(out[b], good[b]), (bad, b)
