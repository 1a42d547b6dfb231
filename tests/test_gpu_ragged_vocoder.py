"""GPU: ragged batches (per-utterance lengths) through every vocoder layer and the public Generator / vocoder_infer interface.

The contract (include/fs2b200.h): with lengths, utterance b is computed on its first n_b = clamp(lens[b] * lens_scale, 0, T) rows exactly
as a B = 1 call on those rows would compute it.  So every check here is "rows < n_b of the batched call == the same operator run alone",
bit for bit, with every row at or beyond n_b of the inputs and every output / workspace byte poisoned with NaN beforehand: a single
read outside an utterance would turn its rows into NaN."""
import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, ops, packing, synth, configs
from fastspeech2_b200.hifigan import AttrDict, Generator
from oracle import fs2_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
WAV_TOL = 1e-4
NAN = float("nan")
# fp32 CUDA-core conv: its tile heuristic (conv_simt.cu `small`) looks at B * T and may pick another tile shape for the B = 1 call.
# Every output element is still one fp32 FMA chain in the same (tap, channel) order, so the bits are expected to agree; should a
# future tile shape reorder that chain, the bar is the existing batch-vs-alone bar of the fp32 path.
SIMT_ALONE_BAR = 2e-6


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _poison_rows(x, lens, scale=1):
    """x [B, T, ...] with rows t >= lens[b] * scale set to NaN (a copy)."""
    x = x.clone()
    for b, n in enumerate(lens):
        x[b, min(n * scale, x.shape[1]):] = NAN
    return x


def _check_alone(got, lens, scale, alone, bar=0.0, zero_tail=False):
    """got [B, T, ...] of the ragged call; alone(b, n) -> [1, n, ...] of the same operator on utterance b's first n rows."""
    T = got.shape[1]
    for b, ln in enumerate(lens):
        n = min(ln * scale, T)
        if zero_tail:
            assert torch.equal(got[b, n:], torch.zeros_like(got[b, n:])), b
        if n == 0:
            continue
        want = alone(b, n)[0]
        g = got[b, :n]
        assert torch.isfinite(g).all(), (b, n)
        if bar == 0.0 or not torch.equal(g, want):
            err = (g - want).abs().max().item()
            assert err <= bar, (b, n, err)


# ---------------------------------------------------------------------------------------------------------------- fs2_conv1d
CONV_CASES = [
    # fmt, B, T, Cin, N, taps, dil, pad, lens, lens_scale
    # tile edges (0, 1, 127, 128, 129, T) and a 40000-row utterance: 318 live 128-row tiles, >= 2 work items for every CTA of 132
    ("split3", 6, 40000, 64, 128, 7, 1, 3, (0, 1, 127, 128, 129, 40000), 1),
    ("f8", 6, 40000, 64, 64, 11, 5, 25, (0, 1, 127, 128, 129, 40000), 1),
    ("split3", 3, 700, 256, 256, 3, 1, 1, (129, 700, 1), 1),                  # two channel blocks (NB = 128)
    ("f8", 3, 2048, 128, 128, 7, 3, 9, (17, 0, 256), 8),                       # lengths in mel frames, 8 rows per frame
    ("simt", 6, 3000, 64, 64, 7, 1, 3, (0, 1, 127, 128, 129, 3000), 1),
    ("simt", 3, 2048, 128, 96, 11, 5, 25, (17, 0, 256), 8),
]


def _conv(fmt, x, w, wt, bias, res, lens, scale, pad, dil, out=None):
    backend = L.CONV_SIMT if fmt == "simt" else L.CONV_TC
    return ops.conv1d(x, w, bias, dilation=dil, pad_left=pad, in_act=L.ACT_LRELU, in_slope=0.1, out_act=L.ACT_LRELU, out_slope=0.1,
                      res=res, alpha=0.5, out=out, w_tc=None if fmt == "simt" else wt, backend=backend, tc_variant=int(fmt == "f8"),
                      x_lens=lens, lens_scale=scale)


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv1d_ragged_equals_each_utterance_alone(case):
    fmt, B, T, Cin, N, taps, dil, pad, lens, scale = case
    x = rnd(B, T, Cin, seed=1, scale=2.0)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias, res = rnd(N, seed=3, scale=0.1), rnd(B, T, N, seed=4)
    wt = packing.pack_conv_tc(w, f8=fmt == "f8").to(DEV) if fmt != "simt" else None
    xd, wd, bd = x.to(DEV), w.to(DEV), bias.to(DEV)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    y = torch.full((B, T, N), NAN, device=DEV)
    _conv(fmt, _poison_rows(x, lens, scale).to(DEV), wd, wt, bd, _poison_rows(res, lens, scale).to(DEV), lens_d, scale, pad, dil, out=y)
    alone = lambda b, n: _conv(fmt, xd[b:b + 1, :n], wd, wt, bd, res[b:b + 1, :n].to(DEV), None, 1, pad, dil)
    torch.cuda.synchronize()
    _check_alone(y, lens, scale, alone, bar=SIMT_ALONE_BAR if fmt == "simt" else 0.0)


@pytest.mark.parametrize("fmt", ["split3", "f8", "simt"])
def test_conv_transpose_phase_groups_ragged(fmt):
    """ConvTranspose1d(k = 2u) as the vocoder runs it: two 2-tap phase groups writing strided column halves of [B][T][u * C_out].
    Input and output rows share n_b."""
    u, C, Co, T, scale = 8, 128, 64, 2000, 8
    lens = (0, 16, 250, 1, 137)
    B = len(lens)
    x = rnd(B, T, C, seed=5, scale=2.0)
    xp, xd = _poison_rows(x, lens, scale).to(DEV), x.to(DEV)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    groups = []
    for g in range(2):
        w = rnd(2, C, (u // 2) * Co, seed=6 + g, scale=(2 * C) ** -0.5)
        groups.append((w.to(DEV), packing.pack_conv_tc(w, f8=fmt == "f8").to(DEV) if fmt != "simt" else None,
                       rnd((u // 2) * Co, seed=8 + g, scale=0.1).to(DEV), 1 - g))

    def run(xx, lens_t, y):
        for g, (w, wt, b, pad) in enumerate(groups):
            ops.conv1d(xx, w, b, pad_left=pad, in_act=L.ACT_LRELU, in_slope=0.1, out=y[:, :, g * (u // 2) * Co:(g + 1) * (u // 2) * Co],
                       w_tc=wt, backend=L.CONV_SIMT if fmt == "simt" else L.CONV_TC, tc_variant=int(fmt == "f8"), x_lens=lens_t,
                       lens_scale=scale)
        return y
    got = run(xp, lens_d, torch.full((B, T, u * Co), NAN, device=DEV))
    alone = lambda b, n: run(xd[b:b + 1, :n], None, torch.empty(1, n, u * Co, device=DEV))
    torch.cuda.synchronize()
    _check_alone(got, lens, scale, alone, bar=SIMT_ALONE_BAR if fmt == "simt" else 0.0)


# ---------------------------------------------------------------------------------------------------------------- fs2_resstack
def _resstack_weights(C, kernels, dils, seed):
    t1, b1, t2, b2 = [], [], [], []
    for j, k in enumerate(kernels):
        t1.append([]); b1.append([]); t2.append([]); b2.append([])
        for d in range(len(dils[j])):
            s = seed + 10 * j + d
            t1[j].append(packing.pack_conv_tc(packing.conv_w(rnd(C, C, k, seed=s, scale=0.6 * (C * k) ** -0.5)), f8=True).to(DEV))
            t2[j].append(packing.pack_conv_tc(packing.conv_w(rnd(C, C, k, seed=s + 500, scale=0.6 * (C * k) ** -0.5)), f8=True).to(DEV))
            b1[j].append(rnd(C, seed=s + 1000, scale=0.05).to(DEV)); b2[j].append(rnd(C, seed=s + 1500, scale=0.05).to(DEV))
    return t1, b1, t2, b2


SHIPPED = ((3, 7, 11), ((1, 3, 5),) * 3)
RESSTACK_CASES = [
    # C, N, kernels, dilations, lens, lens_scale, accumulate      (output rows per work item: 392 at C = 32, 136 at C = 64)
    (32, 3000, *SHIPPED, (0, 1, 391, 392, 393, 3000), 1, False),
    (64, 40000, *SHIPPED, (0, 1, 135, 136, 137, 40000), 1, False),    # 300 live tiles: >= 2 work items for every CTA of 132
    (64, 4096, *SHIPPED, (3, 16, 0), 256, False),                      # lengths in mel frames, 256 rows per frame
    (64, 20000, (3,), ((5,),), (0, 1, 135, 137, 20000, 9999), 1, True),  # per-pair mode: y += alpha * pair(x)
    (32, 20000, (3,), ((1,),), (391, 20000, 0, 393), 1, False),
]


@pytest.mark.parametrize("case", RESSTACK_CASES)
def test_resstack_ragged_equals_each_utterance_alone(case):
    C, N, kernels, dils, lens, scale, acc = case
    B = len(lens)
    t1, b1, t2, b2 = _resstack_weights(C, kernels, dils, seed=60)
    x, y0 = rnd(B, N, C, seed=61, scale=1.5), rnd(B, N, C, seed=62)
    alpha = 1.0 / 3 if acc else 0.0
    out = _poison_rows(y0, lens, scale).to(DEV) if acc else torch.full((B, N, C), NAN, device=DEV)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ops.resstack(_poison_rows(x, lens, scale).to(DEV), kernels, dils, t1, b1, t2, b2, alpha=alpha, out=out, accumulate=acc,
                 lens=lens_d, lens_scale=scale)
    xd = x.to(DEV)
    alone = lambda b, n: ops.resstack(xd[b:b + 1, :n].contiguous(), kernels, dils, t1, b1, t2, b2, alpha=alpha,
                                      out=y0[b:b + 1, :n].to(DEV).contiguous() if acc else None, accumulate=acc)
    torch.cuda.synchronize()
    _check_alone(out, lens, scale, alone)


# ---------------------------------------------------------------------------------------------------------------- fs2_conv_post
@pytest.mark.parametrize("C", [32, 16])     # 32: the generator's shape (register kernel); 16: the staged generic kernel
def test_conv_post_ragged_zero_tail(C):
    T, scale = 256 * 40, 256
    lens = (0, 1, 3, 40, 17)
    B = len(lens)
    x = rnd(B, T, C, seed=70)
    w, bias = rnd(7, C, seed=71, scale=C ** -0.5).to(DEV), rnd(1, seed=72, scale=0.1).to(DEV)
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV)
    got = ops.conv_post(_poison_rows(x, lens, scale).to(DEV), w, bias, lens=lens_d, lens_scale=scale)
    xd = x.to(DEV)
    alone = lambda b, n: ops.conv_post(xd[b:b + 1, :n].contiguous(), w, bias)
    torch.cuda.synchronize()
    _check_alone(got, lens, scale, alone, zero_tail=True)
    # clamped, never trusted: negative and beyond-T device lengths behave as 0 and T
    odd = ops.conv_post(xd[:2].contiguous(), w, bias, lens=torch.tensor([-5, 10 ** 6], dtype=torch.int32, device=DEV), lens_scale=scale)
    torch.cuda.synchronize()
    assert torch.equal(odd[0], torch.zeros_like(odd[0])) and torch.equal(odd[1], ops.conv_post(xd[1:2].contiguous(), w, bias)[0])


# ---------------------------------------------------------------------------------------------------------------- Generator
def _generator(seed, sd=None):
    h = AttrDict(configs.HIFIGAN_CONFIG)
    sd = synth.hifigan_state_dict(h, seed=seed) if sd is None else sd
    gen = Generator(h)
    gen.load_state_dict(sd)
    gen.eval()
    gen.remove_weight_norm()
    return gen.to(DEV), sd


def _ragged_poisoned(gen, mel, lens):
    """gen(mel, mel_lens) with the padded mel frames and the whole workspace filled with NaN before the timed call."""
    mel = mel.clone()
    for b, n in enumerate(lens):
        mel[b, :, n:] = NAN
    mel_d = mel.to(DEV)
    gen(mel_d, mel_lens=torch.tensor(lens))             # allocates the workspace for this shape
    gen._ws.fill_(0xFF)                                  # every fp32 word = NaN
    return gen(mel_d, mel_lens=torch.tensor(lens))


def _check_generator(gen, sd, mel, lens, bar_alone=0.0, oracle=True):
    got = _ragged_poisoned(gen, mel, lens)
    torch.cuda.synchronize()
    assert got.shape == (len(lens), 1, 256 * mel.shape[2])
    errs = []
    for b, n in enumerate(lens):
        assert torch.equal(got[b, :, 256 * n:], torch.zeros_like(got[b, :, 256 * n:])), b
        if n == 0:
            continue
        alone = gen(mel[b:b + 1, :, :n].to(DEV))[0]
        g = got[b, :, :256 * n]
        assert torch.isfinite(g).all(), b
        if not torch.equal(g, alone):
            assert (g - alone).abs().max().item() <= bar_alone, (b, n)
        if oracle:
            errs.append((g.cpu() - O.hifigan_forward(sd, mel[b:b + 1, :, :n])[0]).abs().max().item())
    assert not errs or max(errs) < WAV_TOL, errs
    return got


POLICIES = {
    "default": {},
    "fused_64ch_stage": {"fused_mask": 0b1100},
    "no_pairs": {"pair_mask": 0},
    "split3_everywhere": {"f8_mask": 0},
    "fp32_cuda_cores": {"use_tensor_cores": False},
}


@pytest.mark.parametrize("policy", list(POLICIES))
def test_generator_ragged_batch_vs_oracle_alone(policy):
    gen, sd = _generator(seed=3)
    for k, v in POLICIES[policy].items():
        setattr(gen, k, v)
    gen._invalidate()
    lens = (60, 0, 1, 9, 33, 47)
    mel = synth.make_mel(len(lens), 60, seed=12)
    _check_generator(gen, sd, mel, lens, bar_alone=SIMT_ALONE_BAR if policy == "fp32_cuda_cores" else 0.0)


def test_generator_all_lengths_full_equals_padded_path():
    gen, _ = _generator(seed=3)
    mel = synth.make_mel(3, 77, seed=13).to(DEV)
    padded = gen(mel)
    ragged = gen(mel, mel_lens=torch.full((3,), 77, dtype=torch.long, device=DEV))
    torch.cuda.synchronize()
    assert torch.equal(padded, ragged)


def test_generator_mel_lens_argument_checks():
    gen, _ = _generator(seed=3)
    mel = synth.make_mel(2, 20, seed=14).to(DEV)
    for bad in (torch.tensor([21, 3]), torch.tensor([-1, 3]), torch.tensor([3.0, 4.0]), torch.tensor([3])):
        with pytest.raises(ValueError):
            gen(mel, mel_lens=bad)
    # device values are clamped by the kernels, not checked on the host
    got = gen(mel, mel_lens=torch.tensor([10 ** 6, -4], dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    assert torch.equal(got[0], gen(mel[:1])[0]) and torch.equal(got[1], torch.zeros_like(got[1]))


def test_generator_ragged_full_size_configs3(libri_configs):
    """BASELINE configs[3] inputs (LibriTTS, B = 64, 64-256 phonemes) run free through FastSpeech2, then the ragged vocoder on out[9]:
    the shortest, the first and the last utterance against the oracle alone and against the GPU alone-run."""
    from fastspeech2_b200.model import FastSpeech2
    pc, mc = libri_configs
    m = FastSpeech2(pc, mc)
    m.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=9))
    m = m.to(DEV).eval()
    gen, sd = _generator(seed=3)
    spk, texts, lens, Lm = synth.make_batch(64, 256, seed=11, n_speakers=904, min_len=64)
    with torch.no_grad():
        out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm)
    mel = out[1].transpose(1, 2)
    got = gen(mel, mel_lens=out[9])
    torch.cuda.synchronize()
    ml = out[9].cpu().tolist()
    assert got.shape == (64, 1, 256 * mel.shape[2])
    for b in sorted({int(np.argmin(ml)), 0, 63}):
        n = ml[b]
        alone = gen(mel[b:b + 1, :, :n])
        assert torch.equal(got[b:b + 1, :, :256 * n], alone), b
        assert torch.equal(got[b, :, 256 * n:], torch.zeros_like(got[b, :, 256 * n:])), b
        err = (alone.cpu() - O.hifigan_forward(sd, mel[b:b + 1, :, :n].cpu())).abs().max().item()
        assert err < WAV_TOL, (b, n, err)


@pytest.mark.parametrize("name", ["LJSpeech", "universal"])
def test_generator_ragged_real_checkpoint(name):
    import os
    from oracle import real_ckpt
    sd = real_ckpt.load(name)
    if sd is None:
        pytest.skip("oracle/_ref/ real-checkpoint fixture not in this snapshot")
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"hifigan_real_{name}.npz"))
    gold = torch.from_numpy(z["mel"])[:1]
    Tg = gold.shape[2]
    starts, lens = (0, Tg // 3, Tg // 5), (Tg, Tg - Tg // 3, Tg // 2)
    mel = torch.zeros(3, 80, Tg)
    for b, (s, n) in enumerate(zip(starts, lens)):
        mel[b, :, :n] = gold[0, :, s:s + n]
    gen, _ = _generator(seed=0, sd=sd)
    _check_generator(gen, sd, mel, lens)


def test_vocoder_infer_ragged_equals_each_utterance_alone(lj_configs):
    from fastspeech2_b200 import dropin
    pc, mc = lj_configs
    gen, _ = _generator(seed=3)
    mel_lens = torch.tensor([40, 7, 0, 23])
    mel = synth.make_mel(4, 40, seed=15)
    for b, n in enumerate(mel_lens.tolist()):
        mel[b, :, n:] = NAN                                   # never read in ragged mode
    hop = pc["preprocessing"]["stft"]["hop_length"]
    lengths = (mel_lens * hop).to(DEV)
    wavs = dropin.vocoder_infer(mel.to(DEV), gen, mc, pc, lengths=lengths, ragged=True)
    scale = pc["preprocessing"]["audio"]["max_wav_value"]
    for b, n in enumerate(mel_lens.tolist()):
        assert wavs[b].dtype.name == "int16" and wavs[b].shape == (n * hop,)
        if n:
            want = (gen(mel[b:b + 1, :, :n].to(DEV)).cpu().numpy() * scale).astype("int16")[0, 0]
            assert (wavs[b] == want).all(), b
    with pytest.raises(ValueError):
        dropin.vocoder_infer(mel.to(DEV), gen, mc, pc, lengths=None, ragged=True)
    with pytest.raises(ValueError):
        dropin.vocoder_infer(mel.to(DEV), gen, mc, pc, lengths=lengths + 1, ragged=True)
