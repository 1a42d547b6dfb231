"""GPU: pools of the eight generators of tests/generator_cases.py (every weight-scale header, tile and bias differs between every pair of
them), at the pool sizes that put the multi-generator kernels into the plans large pools pick: every stream bit for bit against its own
generator's forward, and each generator's stream against the fp32 CPU oracle of its rescaled state dict.

The pool sizes are the ones tests/test_stream_multi_plans_cpu.py checks on 132 and 114 SMs; here the device's own SM count plans them
again and each pool is asserted to reach its plans before it runs: the tensor-core conv at NG >= 2 (V2's ups 0 phase groups, V1's
per-layer ResBlock convs) with CTAs of more than 16 units whose consecutive items change generator, every fused ResBlock launch with a
CTA that runs consecutive items of different generators, and the exact kernels at 64- and 128-row tiles."""
import pytest
import torch

from fastspeech2_b200 import synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from oracle import fs2_oracle as O
from tests import generator_cases as GC
from tests.test_gpu_conv_groups import device_sms
from tests.test_gpu_resample_mixed import _offline
from tests.test_gpu_stream_multi import _run

pytestmark = pytest.mark.gpu
DEV = "cuda"
WAV_TOL = 1e-4                                         # the generator-vs-oracle bar of V1 (tests/test_gpu_model.py) and V2 (WAV_TOL)


def _generators(cfg, policy):
    """The 8 generators of cfg under policy, on the GPU (loaded as a checkpoint is: weight norm folded after loading)."""
    out = []
    for sd in GC.state_dicts(cfg):
        g = Generator(AttrDict(GC.CFGS[cfg]))
        g.load_state_dict(sd)
        g.eval()
        g.remove_weight_norm()
        for k, v in GC.POLICIES[policy].items():
            setattr(g, k, v)
        g._invalidate()
        out.append(g.to(DEV))
    return out


def _check_plans(ks, tc):
    """The plan facts of one pool on this device (tests/test_stream_multi_plans_cpu.py checks them on 132 and 114 SMs)."""
    for k in ks:
        if k["kernel"] == "resstack":
            assert GC.switches(k["seq"], k["grid"]) > 0, k["name"]
    if tc:
        conv = [k for k in ks if k["kernel"] == "conv_tc"]
        assert any(k["NG"] >= 2 for k in conv)
        assert any(k["units"] > GC.G.SLOTS and GC.switches(k["seq"], k["grid"]) > 0 for k in conv)


@pytest.mark.parametrize("cfg_policy", GC.CFG_POLICIES, ids=[f"{c}-{p}" for c, p in GC.CFG_POLICIES])
def test_pool_of_eight_generators_equals_each_forward(cfg_policy):
    cfg, policy = cfg_policy
    gens = _generators(cfg, policy)
    m, tc = GC.model_of(cfg, policy)
    packed = gens[0]._packed[0] if gens[0]._packed else gens[0]._pack()[0]
    assert (packed.f8_mask, packed.fused_mask, packed.pair_mask) == (m.f8_mask, m.fused_mask, m.pair_mask)
    for n in GC.POOLS[(cfg, policy)]:
        lens = GC.pool_lens(n)
        if n == max(GC.POOLS[(cfg, policy)]):
            _check_plans(GC.launch_kernels(m, tc, n, lens, [0] * n, GC.CHUNK, device_sms()), tc)
        pool = gens[0].stream_pool(chunk_frames=GC.CHUNK, generators=gens[1:])
        mels = [synth.make_mel(1, t, seed=2000 + b)[0].to(DEV) for b, t in enumerate(lens)]
        which = [GC.gen_of(b) for b in range(n)]
        out = _run(pool, mels, which, [0] * n)
        for b, mel in enumerate(mels):
            assert torch.equal(out[b], gens[which[b]](mel[None])), (n, b, which[b])


@pytest.mark.parametrize("cfg", sorted(GC.CFGS))
def test_mixed_pool_of_eight_generators_added_and_open_streams_and_formats(cfg):
    """Added and open streams of all 8 generators, fed block by block, at the generator's rate in fp32, resampled, PCM16 and mu-law."""
    gens = _generators(cfg, "default")
    pool = gens[0].stream_pool(chunk_frames=GC.CHUNK, generators=gens[1:])
    spec = [(70, 5, None, None, "add"), (45, 2, 16000, "pcm16", "open"), (90, 7, 8000, "ulaw", "add"), (33, 0, 24000, "f32", "open"),
            (61, 3, None, None, "open"), (12, 6, 16000, "pcm16", "add"), (52, 1, None, "pcm16", "open"), (38, 4, None, None, "add"),
            (80, 5, 16000, "f32", "open")]
    mels = [synth.make_mel(1, n, seed=3000 + k)[0].to(DEV) for k, (n, *_rest) in enumerate(spec)]
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
                step = min(5 + 4 * k, spec[k][0] - fed[k])
                pool.feed(h, mels[k][:, fed[k]:fed[k] + step])
                fed[k] += step
                if fed[k] == spec[k][0]:
                    pool.close(h)
        for h, first, chunk in pool.step():
            parts.setdefault(handles[h], []).append(chunk.reshape(-1))
        tick += 1
        assert tick < 200
    for k, (n, g, rate, enc, kind) in enumerate(spec):
        got = torch.cat(parts[k])
        if rate is None and enc in (None, "f32"):
            assert torch.equal(got, gens[g](mels[k][None]).reshape(-1)), k
        else:
            assert torch.equal(got, _offline(gens[g], mels[k], rate or 22050, enc or "f32").reshape(-1)), k


@pytest.mark.parametrize("cfg", sorted(GC.CFGS))
def test_each_generators_stream_against_the_oracle(cfg, parity_log):
    """One stream per generator in one pool: its joined chunks within WAV_TOL of the fp32 oracle of that generator's rescaled state
    dict, which catches a fault the pool and forward would share (a packing error at an unusual scale)."""
    gens = _generators(cfg, "default")
    pool = gens[0].stream_pool(chunk_frames=GC.CHUNK, generators=gens[1:])
    lens = [41 + 7 * k for k in range(GC.MAX_GENERATORS)]
    mels = [synth.make_mel(1, n, seed=4000 + k)[0] for k, n in enumerate(lens)]
    which = [GC.gen_of(b) for b in range(GC.MAX_GENERATORS)]
    out = _run(pool, [mel.to(DEV) for mel in mels], which, [0, 1, 0, 2, 0, 1, 0, 0])
    worst = 0.0
    for b, mel in enumerate(mels):
        want = O.hifigan_forward(GC.state_dicts(cfg)[which[b]], mel[None], **GC.oracle_kwargs(cfg))
        err = (out[b].cpu() - want).abs().max().item()
        peak = want.abs().max().item()
        parity_log("test_each_generators_stream_against_the_oracle", cfg=cfg, generator=which[b], err=err, peak=peak, bar=WAV_TOL,
                   frac=err / WAV_TOL)
        worst = max(worst, err)
        assert err < WAV_TOL and peak > 0.05, (b, which[b], err, peak)
    print(f"{cfg}: worst oracle error {worst:.3e} = {worst / WAV_TOL:.2f} of the bar")
