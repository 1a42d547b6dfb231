"""GPU: NaN, Inf and extreme values stay inside the utterance, stream and model they belong to.

Every "equals each utterance alone" test elsewhere runs finite data, on which a kernel that reads a neighbour's rows (or another
model's weights) and cancels them with a zero gives the right bits.  Here one tenant is poisoned (tests/isolation_cases.py: NaN, +-Inf,
65504 and 3e38 at its first, last and tile / chunk-boundary rows, in a whole frame or one channel, first, middle or last in the batch)
and, with `same` (NaN masks, infinities, finite bits) as the bar:
  A. activation side: every other tenant equals the clean run, and the poisoned one equals its own solo call with the same poison;
  B. weight side: a pool or bank with one poisoned model gives every other model's tenants that model's own output bit for bit;
  C. the NaN cone: one NaN frame or channel gives a waveform whose NaN mask is the fp64 oracle's, and the clean run's bits elsewhere;
  D. the conversion epilogue's encodings of NaN and +-Inf.
A solo call is B = 1 where the kernels' plan does not depend on B; where it may (the exact fp32 kernels pick tiles from B * T), it is a
batch of the same shape holding the poisoned tenant's input alone, in every row."""
import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, ops, packing, synth
from fastspeech2_b200.hifigan import AttrDict
from fastspeech2_b200.model import FastSpeech2, VoiceBank
from fastspeech2_b200.resample import ENCODINGS, Resampler, design_taps
from oracle import fs2_oracle as O
from oracle.resample_ref import resample_ref
from tests import isolation_cases as I
from tests.isolation_cases import NAN, POISONS, diff, same
from tests.test_gpu_resample_mixed import _offline
from tests.test_gpu_stream_multi import POLICIES, _run as _run_multi
from tests.test_gpu_stream_vocoder import _generator
from tests.test_resample_mixed_cpu import g711_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
CFG_POLICIES = [(c, p) for c in sorted(CFGS) for p in sorted(POLICIES) if not (p == "wide_pairs" and c != "v1")]


def rnd(*shape, seed=0, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


def _assert_isolated(got, clean, b, solo, part, what):
    """Tenant b of got equals solo, every other tenant equals its clean output; part(t, c) is tenant c's compared slice of t."""
    for c in range(clean.shape[0]):
        if c != b:
            g, w = part(got, c), part(clean, c)
            assert same(g, w), f"{what}: tenant {c} changed by the poison in tenant {b}: {diff(g, w)}"
    g = part(got, b)
    assert same(g, solo), f"{what}: poisoned tenant {b} differs from its solo call: {diff(g, solo)}"


def _sweep(run, x, n_of, boundary, solo, part, what, axis=1, poisons=tuple(POISONS)):
    """run(x) -> [B, ...]; solo(xp, b) -> tenant b's output alone, compared to part(run(xp), b)."""
    clean = run(x)
    for name, b, place, row in I.cases(x.shape[0], n_of, boundary, poisons):
        xp = I.poison(x, b, row, POISONS[name], place, axis=axis, channel=5)
        _assert_isolated(run(xp), clean, b, solo(xp, b), part, f"{what} {name} at {place} row {row}")


# ============================================================================================ A. activation side: the ops
# fmt, B, T, Cin, N, taps, dil, pad.  The padded batches (no lengths) hold several 128-row tiles per utterance and >= 2 work items per
# CTA of 132, so a tile's halo row past an utterance's last row is the next utterance's row 0 in memory.
CONV_CASES = {
    "split3": (3, 12800, 64, 128, 7, 1, 3),
    "f8": (3, 12800, 64, 64, 11, 5, 25),
    "segmented": (3, 6000, 256, 256, 3, 1, 1),
    "simt": (3, 3000, 64, 64, 7, 1, 3),
}


def _conv_run(fmt, w, wt, bias, res, dil, pad, lens=None):
    variant = {"split3": 0, "f8": 1, "segmented": 2 | 4, "simt": 0}[fmt]
    seg = fmt == "segmented"                           # as the encoder runs it: input ReLU (a slope-0 LeakyReLU), residual, no output act

    def run(x, lens=lens, res=res):
        return ops.conv1d(x, w, bias, dilation=dil, pad_left=pad, in_act=L.ACT_LRELU, in_slope=0.0 if seg else 0.1,
                          out_act=L.ACT_NONE if seg else L.ACT_LRELU, out_slope=0.1, res=res, alpha=1.0 if seg else 0.5, w_tc=wt,
                          backend=L.CONV_SIMT if fmt == "simt" else L.CONV_TC, tc_variant=variant, x_lens=lens)
    return run


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("fmt", sorted(CONV_CASES))
def test_conv1d(fmt, ragged):
    B, T, Cin, N, taps, dil, pad = CONV_CASES[fmt]
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    wt = None if fmt == "simt" else (packing.pack_conv_tc_segments(w.cpu()) if fmt == "segmented" else
                                     packing.pack_conv_tc(w.cpu(), f8=fmt == "f8")).to(DEV)
    bias, res = rnd(N, seed=3, scale=0.1), rnd(B, T, N, seed=4)
    x = rnd(B, T, Cin, seed=1, scale=2.0)
    lens = [T, T - 1 - 3 * I.TILE, I.TILE + 1] if ragged else [T] * B
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV) if ragged else None
    run = _conv_run(fmt, w, wt, bias, res, dil, pad, lens_d)
    part = lambda t, c: t[c, :lens[c]]
    if fmt == "simt":           # the fp32 kernel's tile depends on B * T: the solo call is a batch of the tenant alone
        solo = lambda xp, b: run(xp[b:b + 1].expand(B, -1, -1).contiguous(), res=res[b:b + 1].expand(B, -1, -1).contiguous(),
                                 lens=None if lens_d is None else lens_d[b:b + 1].expand(B).contiguous())[0, :lens[b]]
    else:
        solo = lambda xp, b: run(xp[b:b + 1, :lens[b]].contiguous(), lens=None, res=res[b:b + 1, :lens[b]].contiguous())[0]
    _sweep(run, x, lambda b: lens[b], I.TILE, solo, part, f"conv1d {fmt} {'ragged' if ragged else 'padded'}")


def _resstack_weights(C, kernels, dils, seed):
    tiles = lambda w: (packing.pack_conv_tc_pad16(w) if C == 8 else packing.pack_conv_tc(w, f8=True)).to(DEV)
    t1, b1, t2, b2 = [], [], [], []
    for j, k in enumerate(kernels):
        s = seed + 10 * j
        t1.append([tiles(packing.conv_w(rnd(C, C, k, seed=s + d, scale=0.6 * (C * k) ** -0.5).cpu())) for d in range(len(dils[j]))])
        t2.append([tiles(packing.conv_w(rnd(C, C, k, seed=s + d + 500, scale=0.6 * (C * k) ** -0.5).cpu())) for d in range(len(dils[j]))])
        b1.append([rnd(C, seed=s + d + 1000, scale=0.05) for d in range(len(dils[j]))])
        b2.append([rnd(C, seed=s + d + 1500, scale=0.05) for d in range(len(dils[j]))])
    return t1, b1, t2, b2


# C -> rows per utterance: each more than two output tiles (136 rows at 64 channels, 392 at 32, 896 at 16 and 8)
RESSTACK_ROWS = {64: 2000, 32: 2400, 16: 4000, 8: 4000}


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("C", sorted(RESSTACK_ROWS))
def test_resstack(C, ragged):
    """fs2_resstack at every width it serves (the 128-channel pairs run in the generator tests under the wide_pairs policy)."""
    kernels, dils = (3, 7, 11), ((1, 3, 5),) * 3
    N, B = RESSTACK_ROWS[C], 3
    ws = _resstack_weights(C, kernels, dils, seed=60)
    x = rnd(B, N, C, seed=61, scale=1.5)
    lens = [N, N - 301, 137] if ragged else [N] * B
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV) if ragged else None
    run = lambda xx, ll=lens_d: ops.resstack(xx.contiguous(), kernels, dils, *ws, lens=ll)
    boundary = {64: 136, 32: 392, 16: 896, 8: 896}[C]
    _sweep(run, x, lambda b: lens[b], boundary, lambda xp, b: run(xp[b:b + 1, :lens[b]], None)[0], lambda t, c: t[c, :lens[c]],
           f"resstack C={C}")


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("C", [32, 16])       # 32: the generator's register kernel; 16: the staged generic kernel
def test_conv_post(C, ragged):
    T, scale, B = 256 * 24, 256, 3
    x = rnd(B, T, C, seed=70)
    w, bias = rnd(7, C, seed=71, scale=C ** -0.5), rnd(1, seed=72, scale=0.1)
    frames = [24, 11, 3] if ragged else [24] * B
    lens = [f * scale for f in frames]
    lens_d = torch.tensor(frames, dtype=torch.int32, device=DEV) if ragged else None
    run = lambda xx, ll=lens_d: ops.conv_post(xx.contiguous(), w, bias, lens=ll, lens_scale=scale)
    _sweep(run, x, lambda b: lens[b], 2 * I.TILE, lambda xp, b: run(xp[b:b + 1, :lens[b]], None)[0], lambda t, c: t[c, :lens[c]],
           f"conv_post C={C}")


@pytest.mark.parametrize("backend", [0, 2])
def test_attention(backend):
    T = 300
    lens = [300, 257, 130]
    qkv = rnd(len(lens), T, 768, seed=3)
    kl = torch.tensor(lens, dtype=torch.int32, device=DEV)
    run = lambda q, k=kl: ops.attention(q.contiguous(), 2, k, backend=backend)
    solo = lambda q, b: run(q[b:b + 1], kl[b:b + 1])[0, :lens[b]]
    _sweep(run, qkv, lambda b: lens[b], I.TILE, solo, lambda t, c: t[c, :lens[c]], f"attention backend {backend}")


def test_layernorm():
    B, T, C = 3, 300, 256
    x, gm, bt = rnd(B, T, C, seed=80), rnd(C, seed=81), rnd(C, seed=82)
    lens = [300, 129, 17]
    ld = torch.tensor(lens, dtype=torch.int32, device=DEV)
    run = lambda xx, ll=ld: ops.layernorm(xx.contiguous(), gm, bt, ll)
    _sweep(run, x, lambda b: lens[b], I.TILE, lambda xp, b: run(xp[b:b + 1], ld[b:b + 1])[0, :lens[b]],
           lambda t, c: t[c, :lens[c]], "layernorm")


@pytest.mark.parametrize("ragged", [False, True])
def test_resample(ragged):
    rs = Resampler(22050, 16000)
    B, N = 3, 9000
    x = rnd(B, N, seed=90, scale=0.3)
    lens = [N, 5000, 700] if ragged else [N] * B
    outs = [rs.n_out(n) for n in lens]
    run = lambda xx, ll=(lens if ragged else None): rs(xx, None if ll is None else torch.tensor(ll, device=DEV))
    _sweep(run, x[:, None], lambda b: lens[b], 4096, lambda xp, b: rs(xp[b:b + 1, :, :lens[b]].contiguous())[0, 0],
           lambda t, c: t[c, 0, :outs[c]], "resample", axis=2)


def _mixed_records(xs, specs, j1s):
    return [(0, x.data_ptr(), 0, 0, x.numel(), x.numel(), 0, j1, Resampler(22050, rate), ENCODINGS[enc])
            for x, (rate, enc), j1 in zip(xs, specs, j1s)]


def test_resample_streams_mixed():
    specs = [(16000, "pcm16"), (8000, "ulaw"), (22050, "f32"), (8000, "alaw"), (24000, "f32")]
    n = [6000, 4000, 5000, 3000, 7000]
    xs = [rnd(k, seed=100 + i, scale=0.3) for i, k in enumerate(n)]
    j1s = [Resampler(22050, r).n_out(k) for (r, _), k in zip(specs, n)]

    def run(xs):
        _, views = Resampler.mixed(_mixed_records(xs, specs, j1s), max(j1s), DEV)
        return [v.clone() for v in views]
    clean = run(xs)
    for name, b, place, row in I.cases(len(xs), lambda b: n[b], 4096):
        xp = list(xs)
        xp[b] = I.poison(xs[b][None], 0, row, POISONS[name], place)[0]
        got = run(xp)
        for c in range(len(xs)):
            want = clean[c] if c != b else _mixed_and_offline(xp[b], *specs[b])
            assert same(got[c], want), (name, b, place, c, diff(got[c], want))


def _mixed_and_offline(x, rate, enc):
    """The offline resampler of x, in enc (G.711 through the numpy oracle of its PCM16)."""
    y = Resampler(22050, rate)(x[None], pcm16=enc != "f32")[0] if rate != 22050 else (ops.wav_to_int16(x[None])[0] if enc != "f32" else x)
    if enc in ("ulaw", "alaw"):
        y = torch.from_numpy(g711_ref(y.cpu().numpy().astype(np.int64), ENCODINGS[enc])).to(DEV)
    return y


# ============================================================================================ A. the vocoder and its pools
MEL_LENS = (64, 41, 23)
FRAME_EDGE = 32          # stage 0's row 256 (a 128-row tile boundary at x8) and a chunk boundary at chunk sizes 1, 16 and 32


def _mel(lens, seed, T=None):
    return synth.make_mel(len(lens), T or max(lens), seed=seed).to(DEV)


def _gen(cfg, policy="default", seed=3, sd=None):
    return _generator(CFGS[cfg], seed=seed, sd=sd, **POLICIES[policy])


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("cfg,policy", CFG_POLICIES)
def test_generator_forward(cfg, policy, ragged):
    gen = _gen(cfg, policy)
    mel = _mel(MEL_LENS, seed=30)
    B, T = mel.shape[0], mel.shape[2]
    lens = list(MEL_LENS) if ragged else [T] * B
    ld = torch.tensor(lens) if ragged else None
    run = lambda m: gen(m, ld)
    # the solo call: the poisoned utterance in every row of a batch of the same shape (the exact kernels' tiles depend on B * T)
    solo = lambda m, b: gen(m[b:b + 1].expand(B, -1, -1), None if ld is None else ld[b:b + 1].expand(B))[0]
    _sweep(run, mel, lambda b: lens[b], FRAME_EDGE, solo, lambda t, c: t[c], f"{cfg} {policy} forward", axis=2)


def _streamed(gen, mel, lens, chunk):
    return torch.cat([w for _, w in gen.stream(mel, mel_lens=lens, chunk_frames=chunk)], dim=2)


@pytest.mark.parametrize("chunk", [1, 32])
@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_generator_stream(cfg, chunk):
    gen = _gen(cfg)
    mel = _mel(MEL_LENS, seed=31)
    ld = torch.tensor(MEL_LENS)
    poisons = ("nan", "+inf", "f32big") if chunk == 1 else tuple(POISONS)
    _sweep(lambda m: _streamed(gen, m, ld, chunk), mel, lambda b: MEL_LENS[b], FRAME_EDGE,
           lambda m, b: gen(m[b:b + 1, :, :MEL_LENS[b]])[0, :, :], lambda t, c: t[c, :, :t.shape[2] * MEL_LENS[c] // mel.shape[2]],
           f"{cfg} stream chunk {chunk}", axis=2, poisons=poisons)


def _pool_run(pool, mels, opened, gens=None, formats=None):
    """Stream k: mels[k] added at tick k % 2, or opened at tick 0 and fed 7 frames a tick (opened[k]); the concatenated chunks."""
    handles, fed, parts, tick = {}, {}, {}, 0
    kw = lambda k: dict(generator=0 if gens is None else gens[k], **({} if formats is None else
                                                                     dict(sample_rate=formats[k][0], encoding=formats[k][1])))
    while tick <= 1 or len(pool):
        for k, m in enumerate(mels):
            if opened[k] and tick == 0:
                handles[pool.open(**kw(k))] = k
                fed[k] = 0
            elif not opened[k] and tick == k % 2:
                handles[pool.add(m, **kw(k))] = k
        for h, k in handles.items():
            if k in fed and fed[k] < mels[k].shape[1]:
                e = min(fed[k] + 7, mels[k].shape[1])
                pool.feed(h, mels[k][:, fed[k]:e])
                fed[k] = e
                if e == mels[k].shape[1]:
                    pool.close(h)
        for h, _first, chunk in pool.step():
            parts.setdefault(handles[h], []).append(chunk.reshape(-1))
        tick += 1
        assert tick < 500
    return [torch.cat(parts[k]) for k in range(len(mels))]


def _pool_sweep(make_pool, mels, opened, alone, what, gens=None, formats=None, poisons=tuple(POISONS)):
    clean = _pool_run(make_pool(), mels, opened, gens, formats)
    for name, b, place, row in I.cases(len(mels), lambda b: mels[b].shape[1], FRAME_EDGE, poisons):
        mp = list(mels)
        mp[b] = I.poison(mels[b][None], 0, row, POISONS[name], place, axis=2)[0]
        got = _pool_run(make_pool(), mp, opened, gens, formats)
        for c in range(len(mels)):
            want = clean[c] if c != b else alone(mp[b], b)
            assert same(got[c], want), f"{what} {name} at {place} row {row} in stream {b}: stream {c}: {diff(got[c], want)}"


@pytest.mark.parametrize("chunk", [1, 32])
@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_stream_pool_added_and_open(cfg, chunk):
    gen = _gen(cfg)
    mels = [_mel((n,), seed=40 + k)[0] for k, n in enumerate((64, 41, 23, 50))]
    opened = [False, True, False, True]
    poisons = ("nan", "-inf", "f16max") if chunk == 1 else tuple(POISONS)
    _pool_sweep(lambda: gen.stream_pool(chunk_frames=chunk), mels, opened, lambda m, b: gen(m[None]).reshape(-1),
                f"{cfg} pool chunk {chunk}", poisons=poisons)


@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_multi_generator_pool_mel(cfg):
    gens = [_gen(cfg, seed=s) for s in (3, 11)]
    mels = [_mel((n,), seed=50 + k)[0] for k, n in enumerate((64, 41, 23, 50))]
    which = [0, 1, 1, 0]
    _pool_sweep(lambda: gens[0].stream_pool(chunk_frames=32, generators=gens[1:]), mels, [False, True, False, False],
                lambda m, b: gens[which[b]](m[None]).reshape(-1), f"{cfg} multi pool", gens=which)


@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_pool_resampling_formats(cfg):
    gen = _gen(cfg)
    formats = [(16000, "pcm16"), (8000, "ulaw"), (8000, "alaw"), (24000, "f32")]
    mels = [_mel((n,), seed=60 + k)[0] for k, n in enumerate((64, 41, 23, 50))]
    _pool_sweep(lambda: gen.stream_pool(chunk_frames=32), mels, [False, False, True, False],
                lambda m, b: _offline(gen, m, *formats[b]).reshape(-1), f"{cfg} pool formats", formats=formats)


# ============================================================================================ A. FastSpeech2
def _fs2(lj_configs, seed=51, tc_mask=None):
    pc, mc = lj_configs
    m = FastSpeech2(pc, mc)
    m.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=seed))
    if tc_mask is not None:
        m.tc_mask = tc_mask
    return m.to(DEV).eval()


def _dev(xs):
    return [x.to(DEV) if torch.is_tensor(x) else x for x in xs]


OUT_NAMES = ("mel", "postnet_mel", "p_pred", "e_pred", "log_d", "d_rounded")


def _check_fs2(out, clean, b, solo, ragged, lens):
    """Rows of the 10-tuple: every utterance but b as in clean, b as in solo (rows up to its lengths in ragged mode)."""
    for i, name in enumerate(OUT_NAMES):
        for c in range(out[0].shape[0]):
            n = int(out[9][c]) if i < 2 else int(lens[c])
            g = out[i][c, :n] if ragged else out[i][c]
            w = (solo[i][0, :n] if ragged else solo[i][c]) if c == b else (clean[i][c, :n] if ragged else clean[i][c])
            assert same(g, w), f"{name} of utterance {c} (poisoned: {b}): {diff(g, w)}"
    assert torch.equal(out[9], clean[9])


@pytest.mark.parametrize("ragged", [False, True])
def test_fastspeech2_pitch_control(lj_configs, ragged):
    model = _fs2(lj_configs)
    spk, texts, lens, Lm = _dev(synth.make_batch(3, 40, seed=70, min_len=12))
    batch = (spk, texts, lens, Lm)
    clean = model(*batch, ragged=ragged)
    T = int(clean[0].shape[1])
    for b in I.positions(3):
        for v in (NAN, float("inf"), -float("inf")):
            pc = torch.ones(3, 1, device=DEV)
            pc[b] = v
            out = model(*batch, ragged=ragged, p_control=pc, max_mel_len=T)
            if ragged:
                n = int(lens[b])
                solo = model(spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n, ragged=True, p_control=pc[b:b + 1])
            else:
                solo = model(*batch, ragged=False, p_control=torch.full((3, 1), v, device=DEV), max_mel_len=T)
            _check_fs2(out, clean, b, solo, ragged, lens)


@pytest.mark.parametrize("ragged", [False, True])
def test_fastspeech2_pitch_energy_targets(lj_configs, ragged):
    model = _fs2(lj_configs)
    spk, texts, lens, Lm = _dev(synth.make_batch(3, 40, seed=71, min_len=12))
    g = torch.Generator().manual_seed(72)
    p_t, e_t = torch.randn(3, Lm, generator=g).to(DEV), torch.randn(3, Lm, generator=g).to(DEV)
    batch = (spk, texts, lens, Lm)
    clean = model(*batch, ragged=ragged, p_targets=p_t, e_targets=e_t)
    T = int(clean[0].shape[1])
    for b in I.positions(3):
        n = int(lens[b])
        for row in (0, n - 1, n // 2):
            pp, ep = p_t.clone(), e_t.clone()
            pp[b, row] = NAN
            ep[b, (row + 1) % n] = NAN
            out = model(*batch, ragged=ragged, p_targets=pp, e_targets=ep, max_mel_len=T)
            if ragged:
                solo = model(spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n, ragged=True, p_targets=pp[b:b + 1, :n],
                             e_targets=ep[b:b + 1, :n])
            else:
                solo = model(*batch, ragged=False, p_targets=pp[b:b + 1].expand(3, -1), e_targets=ep[b:b + 1].expand(3, -1), max_mel_len=T)
            _check_fs2(out, clean, b, solo, ragged, lens)


# ============================================================================================ B. weight side
def _poisoned_generator(cfg, policy, seed, how):
    """A generator whose folded weights are poisoned: 'all' every weight NaN, 'inf' one conv_pre weight +Inf, else the name of the
    bias that gets one NaN channel."""
    gen = _gen(cfg, policy, seed=seed)
    params = dict(gen.named_parameters())
    with torch.no_grad():
        if how == "all":
            for k, p in params.items():
                if k.endswith("weight"):
                    p.fill_(NAN)
        elif how == "inf":
            params["conv_pre.weight"][3, 7, 2] = float("inf")
        else:
            params[how].view(-1)[5 % params[how].numel()] = NAN
    gen._invalidate()
    return gen


def _bias_families(cfg):
    """One bias per layer family: conv_pre, an upsample stage's (both phase groups), a ResBlock conv of a fused stage, a ResBlock conv
    of a per-layer stage under the per_layer policy, and conv_post."""
    h = AttrDict(CFGS[cfg])
    nk = len(h.resblock_kernel_sizes)
    fused_stage = len(h.upsample_rates) - 1
    return ["conv_pre.bias", "ups.1.bias", f"resblocks.{fused_stage * nk + 1}.convs1.2.bias", "resblocks.1.convs2.0.bias", "conv_post.bias"]


@pytest.mark.parametrize("cfg,policy", [("v1", "default"), ("v1", "per_layer"), ("v2", "default"), ("v2", "per_layer")])
def test_multi_generator_pool_poisoned_weights(cfg, policy):
    mels = [_mel((n,), seed=80 + k)[0] for k, n in enumerate((64, 41, 23, 50, 37))]
    which = [0, 1, 2, 1, 0]
    seeds = (3, 11, 17)
    clean = [_gen(cfg, policy, seed=s) for s in seeds]
    own = [clean[g](mels[s][None]) for s, g in enumerate(which)]
    for k in (0, 1, 2):
        for how in ["all", "inf"] + _bias_families(cfg):
            gens = list(clean)
            gens[k] = _poisoned_generator(cfg, policy, seeds[k], how)
            pool = gens[0].stream_pool(chunk_frames=32, generators=gens[1:])
            out = _run_multi(pool, mels, which, [0, 0, 1, 0, 1])
            for s, g in enumerate(which):
                want = gens[k](mels[s][None]) if g == k else own[s]
                assert same(out[s], want), f"{cfg} {policy} generator {k} poisoned ({how}): stream {s} on generator {g}: {diff(out[s], want)}"
                assert g == k or torch.isfinite(want).all()


# tables whose NaN reaches the outputs but not the durations: the decoder side, and the encoder, whose NaN rows the duration
# predictor's input ReLU (fmaxf(v, 0) = 0 for NaN) turns into zeros (DESIGN.md section 3)
TABLES = ("decoder.layer_stack.1.pos_ffn.w_1.weight", "decoder.layer_stack.0.slf_attn.layer_norm.weight", "mel_linear.bias",
          "postnet.convolutions.2.0.conv.weight", "variance_adaptor.pitch_embedding.weight", "variance_adaptor.energy_embedding.weight",
          "encoder.layer_stack.0.slf_attn.layer_norm.weight")
# tables past the duration predictor's last ReLU: a NaN duration
DURATION_TABLES = ("variance_adaptor.duration_predictor.conv_layer.layer_norm_2.bias", "variance_adaptor.duration_predictor.linear_layer.bias")


def _poisoned_voice(lj_configs, seed, key):
    pc, mc = lj_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=seed)
    sd[key] = sd[key].clone()
    if key.endswith("_embedding.weight"):
        sd[key][:] = NAN                               # every bucket's row: whichever the predictions pick
    else:
        sd[key].view(-1)[7 % sd[key].numel()] = NAN
    m = FastSpeech2(pc, mc)
    m.load_state_dict(sd)
    return m.to(DEV).eval()


VOICE = [0, 2, 1, 1, 0, 2, 1]


@pytest.mark.parametrize("key", TABLES)
def test_voice_bank_poisoned_tables(lj_configs, key):
    batch = _dev(synth.make_batch(len(VOICE), 48, seed=90, min_len=8))
    spk, texts, lens, _ = batch
    seeds = (51, 52, 53)
    clean = [_fs2(lj_configs, seed=s) for s in seeds]
    for k in (0, 1, 2):
        models = list(clean)
        models[k] = _poisoned_voice(lj_configs, seeds[k], key)
        out = VoiceBank(models)(torch.tensor(VOICE), *batch, ragged=True)
        for b, v in enumerate(VOICE):
            n = int(lens[b])
            solo = models[v](spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n, ragged=True)
            ml = int(out[9][b])
            assert ml == int(solo[9][0]), (key, k, b)
            for i, name in enumerate(OUT_NAMES):
                g, w = (out[i][b, :ml], solo[i][0]) if i < 2 else (out[i][b, :n], solo[i][0, :n])
                assert same(g, w), f"{key} poisoned in voice {k}: {name} of utterance {b} (voice {v}): {diff(g, w)}"
                if v != k:
                    assert torch.isfinite(g).all(), (key, k, b, name)


@pytest.mark.parametrize("key", DURATION_TABLES)
def test_voice_bank_nan_duration_raises(lj_configs, key):
    """NaN past the duration predictor's last ReLU makes a duration NaN: the bank call raises Fs2Error naming it (the reference raises
    there too), not a CUDA error, and the bank runs clean batches afterwards."""
    batch = _dev(synth.make_batch(len(VOICE), 48, seed=91, min_len=8))
    models = [_poisoned_voice(lj_configs, 52, key) if i == 1 else _fs2(lj_configs, seed=s) for i, s in enumerate((51, 52, 53))]
    bank = VoiceBank(models)
    with pytest.raises(L.Fs2Error, match="NaN"):
        bank(torch.tensor(VOICE), *batch, ragged=True)
    ok = bank(torch.tensor([0, 2, 0, 2, 0, 2, 0]), *batch, ragged=True)
    torch.cuda.synchronize()
    assert torch.isfinite(ok[1]).all()


# ============================================================================================ C. the NaN cone against fp64
CONE_T = {"v1": 48, "v2": 96}
_ORACLE = {}


def _oracle_nan_mask(cfg, sd_seed, mel, key):
    """The NaN mask of the fp64 oracle's waveform of mel [1, 80, n] (CPU), cached by key."""
    if key not in _ORACLE:
        from tests.generator_cases import oracle_kwargs
        h = AttrDict(CFGS[cfg])
        y = O.hifigan_forward(synth.hifigan_state_dict(h, seed=sd_seed), mel.double(), dtype=torch.float64, **oracle_kwargs(cfg))
        _ORACLE[key] = torch.isnan(y[0, 0])
    return _ORACLE[key]


def _intervals(mask):
    idx = mask.nonzero()[:, 0]
    if not len(idx):
        return 0
    return 1 + int((idx[1:] - idx[:-1] > 1).sum())


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("policy", ["default", "exact"])
@pytest.mark.parametrize("cfg", sorted(CFGS))
def test_nan_cone_equals_the_fp64_oracle(cfg, policy, ragged):
    T = CONE_T[cfg]
    lens = [T, T // 2 + 3, T - 9]
    gen = _gen(cfg, policy)
    mel = _mel(lens, seed=33, T=T)
    ld = torch.tensor(lens) if ragged else None
    clean = gen(mel, ld)
    up = clean.shape[-1] // T
    for b in I.positions(3):
        n = lens[b] if ragged else T
        for place, row in (("frame", n // 2), ("channel", 1), ("frame", n - 1), ("channel", min(FRAME_EDGE, n - 2))):
            mp = I.poison(mel, b, row, NAN, place, axis=2, channel=17)
            got = gen(mp, ld)
            want = _oracle_nan_mask(cfg, 3, mp[b:b + 1, :, :n].cpu(), (cfg, b, n, place, row))
            assert _intervals(want) == 1, (cfg, b, place, row)
            g = got[b, 0, :n * up]
            assert torch.equal(torch.isnan(g).cpu(), want), f"{cfg} {policy} {place} {row} in {b}: NaN mask {diff(g.cpu(), want.float())}"
            nan = torch.isnan(got)
            assert int(nan.sum()) == int(want.sum()), "NaN outside the poisoned utterance's cone"
            assert same(torch.where(nan, 0.0, got), torch.where(nan, 0.0, clean)), (cfg, policy, b, place, row)


def test_nan_cone_of_the_resampler_equals_the_fp64_reference():
    for rate in (8000, 16000, 24000, 44100):
        rs = Resampler(22050, rate)
        h = design_taps(rs.up, rs.down)
        B, N = 3, 3000
        x = rnd(B, N, seed=95, scale=0.3)
        lens = torch.tensor([N, 1700, 900])
        clean = rs(x, lens)
        for b in I.positions(B):
            n = int(lens[b])
            for i in (0, n // 2, n - 1):
                xp = x.clone()
                xp[b, i] = NAN
                got = rs(xp, lens)
                want = np.isnan(resample_ref(xp[b, :n].cpu().numpy(), h, rs.up, rs.down))
                assert _intervals(torch.from_numpy(want)) == 1
                m = rs.n_out(n)
                assert np.array_equal(torch.isnan(got[b, :m]).cpu().numpy(), want), (rate, b, i)
                nan = torch.isnan(got)
                assert int(nan.sum()) == int(want.sum()), (rate, b, i)
                assert same(torch.where(nan, 0.0, got), torch.where(nan, 0.0, clean)), (rate, b, i)


# ============================================================================================ D. encodings of non-finite samples
def test_non_finite_samples_encode_as_pinned():
    """NaN converts to PCM 0 (the float-to-int convert maps NaN to 0), so mu-law 0xFF and A-law 0xD5; +-Inf clamp to 32767 / -32768,
    through fs2_wav_to_int16 and through one mixed-format call at the identity ratio and at 16 kHz."""
    v = torch.tensor([NAN, float("inf"), -float("inf"), 0.5, -NAN], device=DEV)
    assert ops.wav_to_int16(v[None]).cpu().tolist()[0] == [0, 32767, -32768, 16384, 0]
    want = {"pcm16": torch.tensor([0, 32767, -32768, 16384, 0], dtype=torch.int16),
            "ulaw": torch.from_numpy(g711_ref(np.array([0, 32767, -32768, 16384, 0]), L.RESAMPLE_ULAW)),
            "alaw": torch.from_numpy(g711_ref(np.array([0, 32767, -32768, 16384, 0]), L.RESAMPLE_ALAW)),
            "f32": v.cpu()}
    assert want["ulaw"][0] == 0xFF and want["alaw"][0] == 0xD5
    encs = list(want)
    _, views = Resampler.mixed(_mixed_records([v] * 4, [(22050, e) for e in encs], [5] * 4), 5, DEV)
    for e, got in zip(encs, views):
        assert same(got.cpu(), want[e]), (e, got.cpu(), want[e])
    # at 16 kHz: a NaN sample gives NaN outputs over its support, and those encode as PCM 0
    x = rnd(2000, seed=96, scale=0.3)
    x[1000] = NAN
    rs = Resampler(22050, 16000)
    f = rs(x[None])[0]
    nan = torch.isnan(f)
    assert bool(nan.any())
    _, views = Resampler.mixed(_mixed_records([x] * 3, [(16000, e) for e in ("pcm16", "ulaw", "alaw")], [rs.n_out(2000)] * 3),
                               rs.n_out(2000), DEV)
    assert (views[0][nan] == 0).all() and (views[1][nan] == 0xFF).all() and (views[2][nan] == 0xD5).all()
    assert torch.equal(views[0][~nan], rs(x[None].nan_to_num(0.0), pcm16=True)[0][~nan])
