"""GPU: HiFi-GAN V2 (configs.HIFIGAN_V2_CONFIG, stages of 64, 32, 16 and 8 channels) through the public Generator against the fp32
oracle and the reference fixture, ragged batches, fs2_resstack at 16 and 8 channels against fp64, and the exact fp32 conv at 8 input
channels."""
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, ops, packing, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from oracle import fs2_oracle as O
from tests import emul_cabi as E
from tests.test_gpu_tc_precision import RESSTACK_C

pytestmark = pytest.mark.gpu
DEV = "cuda"
WAV_TOL = 1e-4
NAN = float("nan")
V2 = AttrDict(configs.HIFIGAN_V2_CONFIG)
GOLD = os.path.join(os.path.dirname(__file__), "golden", "hifigan_v2.npz")


def _generator(seed, **policy):
    sd = synth.hifigan_state_dict(V2, seed=seed)
    gen = Generator(V2)
    gen.load_state_dict(sd)
    gen.eval()
    gen.remove_weight_norm()
    for k, v in policy.items():
        setattr(gen, k, v)
    return gen.to(DEV), sd


# "unfused" still runs the 16-channel stage's k = 3 pairs through fs2_resstack (pair_mask bit 2); "per_layer" runs no ResBlock fused
POLICIES = {"default": {}, "unfused": {"fused_mask": 0}, "per_layer": {"fused_mask": 0, "pair_mask": 0},
            "fp32_cuda_cores": {"use_tensor_cores": False}}


@pytest.mark.parametrize("policy", list(POLICIES))
def test_v2_vs_oracle(policy):
    gen, sd = _generator(5, **POLICIES[policy])
    for B, T in ((1, 1), (1, 7), (2, 50), (3, 129)):
        mel = synth.make_mel(B, T, seed=B * 1000 + T)
        want = O.hifigan_forward(sd, mel)
        got = gen(mel.to(DEV))
        cl = gen(mel.transpose(1, 2).contiguous().to(DEV).transpose(1, 2))     # the channels-last view FastSpeech2's output gives
        torch.cuda.synchronize()
        assert got.shape == want.shape
        assert (got.cpu() - want).abs().max().item() < WAV_TOL, (policy, B, T)
        assert torch.equal(cl, got), (policy, B, T)


def test_v2_reference_fixture():
    z = np.load(GOLD)
    gen, _ = _generator(int(z["seed"]))
    wav = gen(torch.from_numpy(z["mel"]).to(DEV))
    torch.cuda.synchronize()
    assert (wav.cpu() - torch.from_numpy(z["wav"])).abs().max().item() < WAV_TOL


def test_v2_full_size():
    """bench.py configs[2]'s shape, B = 16 x 1012 frames: the first and last rows against the oracle, and the middle row alone against
    the same row of the batch."""
    gen, sd = _generator(7)
    mel = synth.make_mel(16, 1012, seed=8)
    wav = gen(mel.to(DEV))
    mid = gen(mel[8:9].to(DEV))
    torch.cuda.synchronize()
    for b in (0, 15):
        assert (wav[b].cpu() - O.hifigan_forward(sd, mel[b:b + 1])[0]).abs().max().item() < WAV_TOL, b
    assert (mid[0] - wav[8]).abs().max().item() < 2e-6


@pytest.mark.parametrize("policy", list(POLICIES))
def test_v2_ragged_equals_each_utterance_alone(policy):
    gen, sd = _generator(9, **POLICIES[policy])
    lens = (60, 0, 1, 9, 33, 47)
    T = 60
    mel = synth.make_mel(len(lens), T, seed=14)
    poisoned = mel.clone()
    for b, n in enumerate(lens):
        poisoned[b, :, n:] = NAN
    md = poisoned.to(DEV)
    gen(md, mel_lens=torch.tensor(lens))                 # allocates the workspace for this shape
    gen._ws.fill_(0xFF)                                  # every fp32 word = NaN
    got = gen(md, mel_lens=torch.tensor(lens))
    torch.cuda.synchronize()
    for b, n in enumerate(lens):
        assert torch.equal(got[b, :, 256 * n:], torch.zeros_like(got[b, :, 256 * n:])), b
        if n == 0:
            continue
        alone = gen(mel[b:b + 1, :, :n].to(DEV))[0]
        torch.cuda.synchronize()
        g = got[b, :, :256 * n]
        assert torch.isfinite(g).all(), (b, n)
        if not torch.equal(g, alone):       # the exact kernel may pick another tile shape alone (tests/test_gpu_ragged_vocoder.py)
            assert policy == "fp32_cuda_cores" and (g - alone).abs().max().item() <= 2e-6, (b, n)
        if n in (1, T):
            assert (alone.cpu() - O.hifigan_forward(sd, mel[b:b + 1, :, :n])[0]).abs().max().item() < WAV_TOL


# ---------------------------------------------------------------------------------------------------------------- fs2_resstack
def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _tiles(w):
    """fs2_resstack's tiles of a [k][C][C] conv weight: the f8 tiles, zero-padded to 16 x 16 at 8 channels."""
    return (packing.pack_conv_tc_pad16(w) if w.shape[1] == 8 else packing.pack_conv_tc(w, f8=True)).to(DEV)


def _weights(C, kernels, dils, seed):
    w1, b1, w2, b2 = [], [], [], []
    for j, k in enumerate(kernels):
        w1.append([]); b1.append([]); w2.append([]); b2.append([])
        for d in range(len(dils[j])):
            s = seed + 10 * j + d
            w1[j].append(packing.conv_w(rnd(C, C, k, seed=s, scale=0.6 * (C * k) ** -0.5)))
            w2[j].append(packing.conv_w(rnd(C, C, k, seed=s + 500, scale=0.6 * (C * k) ** -0.5)))
            b1[j].append(rnd(C, seed=s + 1000, scale=0.05)); b2[j].append(rnd(C, seed=s + 1500, scale=0.05))
    return w1, b1, w2, b2


GUARD = 1024          # floats of sentinel on each side of y


def _guarded(B, N, C, fill=NAN):
    buf = torch.full((2 * GUARD + B * N * C,), 12345.0, device=DEV)
    y = buf[GUARD:GUARD + B * N * C].view(B, N, C)
    y.fill_(fill)
    return buf, y


def _guards_intact(buf):
    return bool((buf[:GUARD] == 12345.0).all() and (buf[-GUARD:] == 12345.0).all())


SHIPPED = ((3, 7, 11), ((1, 3, 5),) * 3)
# B, N, C, kernels, dilations     (fs2_resstack_plan at 16 and 8 channels: TILE = 896 for the shipped group)
NARROW_CASES = [(B, N, C, *SHIPPED) for C in (16, 8) for B, N in ((2, 1), (2, 50), (2, 895), (1, 896), (2, 897), (6, 40000))]


@pytest.mark.parametrize("case", NARROW_CASES, ids=[f"C{c[2]}_B{c[0]}_N{c[1]}" for c in NARROW_CASES])
def test_resstack_narrow_vs_fp64(case, parity_log):
    """One sample, shorter than the halo, one TILE and TILE +- 1 rows, and 270 work items (>= 2 per CTA of 132): per element against fp64
    within the f16 + f8 bars of test_gpu_tc_precision.resstack_check; no byte of y outside [B][N][C] is written."""
    B, N, C, kernels, dils = case
    x = rnd(B, N, C, seed=21)
    w1, b1, w2, b2 = _weights(C, kernels, dils, seed=100)
    t = lambda ws: [[_tiles(v) for v in row] for row in ws]
    dv = lambda ws: [[v.to(DEV) for v in row] for row in ws]
    buf, y = _guarded(B, N, C)
    ops.resstack(x.to(DEV), kernels, dils, t(w1), dv(b1), t(w2), dv(b2), out=y)
    torch.cuda.synchronize()
    assert _guards_intact(buf)
    got = y.cpu()
    assert torch.isfinite(got).all()
    utts = [0, B - 1] if N > 5000 else list(range(B))          # fp64 on the first and last utterance of the large case
    y64, S, R = E.resstack_contract(x[utts], kernels, dils, w1, b1, w2, b2)
    _, eb = E.tc_errors(got[utts], y64, y64, S, R)
    parity_log("test_resstack_narrow_vs_fp64", C=C, N=N, err_fp64=eb, bar=RESSTACK_C)
    assert eb <= RESSTACK_C, eb


@pytest.mark.parametrize("C", [16, 8])
def test_resstack_narrow_single_pair_accumulate(C):
    """n_kernels = n_dil = 1, accumulate: y += alpha * (conv_k,1(lrelu(conv_k,d(lrelu(x)))) + x), against fp64."""
    B, N, k, d = 2, 2000, 11, 5
    x, y0 = rnd(B, N, C, seed=31), rnd(B, N, C, seed=32)
    w1, b1, w2, b2 = _weights(C, (k,), ((d,),), seed=200)
    buf, y = _guarded(B, N, C)
    y.copy_(y0.to(DEV))
    ops.resstack(x.to(DEV), (k,), ((d,),), [[_tiles(w1[0][0])]], [[b1[0][0].to(DEV)]], [[_tiles(w2[0][0])]], [[b2[0][0].to(DEV)]],
                 alpha=0.5, out=y, accumulate=True)
    torch.cuda.synchronize()
    assert _guards_intact(buf)
    y64, S, R = E.resstack_contract(x, (k,), ((d,),), w1, b1, w2, b2, alpha=0.5, y_prev=y0)
    _, eb = E.tc_errors(y.cpu(), y64, y64, S, R)
    assert eb <= RESSTACK_C, eb


@pytest.mark.parametrize("C", [16, 8])
def test_resstack_narrow_ragged_equals_each_utterance_alone(C):
    lens = (0, 1, 895, 896, 897, 40000)
    B, N = len(lens), 40000
    w1, b1, w2, b2 = _weights(C, *SHIPPED, seed=60)
    t1, t2 = [[_tiles(v) for v in row] for row in w1], [[_tiles(v) for v in row] for row in w2]
    b1, b2 = [[v.to(DEV) for v in row] for row in b1], [[v.to(DEV) for v in row] for row in b2]
    x = rnd(B, N, C, seed=61, scale=1.5)
    xp = x.clone()
    for b, n in enumerate(lens):
        xp[b, n:] = NAN
    buf, y = _guarded(B, N, C)
    ops.resstack(xp.to(DEV), *SHIPPED, t1, b1, t2, b2, out=y, lens=torch.tensor(lens, dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    assert _guards_intact(buf)
    xd = x.to(DEV)
    for b, n in enumerate(lens):
        if n == 0:
            continue
        alone = ops.resstack(xd[b:b + 1, :n].contiguous(), *SHIPPED, t1, b1, t2, b2)
        torch.cuda.synchronize()
        assert torch.equal(y[b, :n], alone[0]), (b, n)


# ---------------------------------------------------------------------------------------------------------------- fs2_conv1d, Cin = 8
@pytest.mark.parametrize("dil,res,acc,ragged", [(1, False, False, False), (5, True, False, False), (3, True, True, False),
                                                 (1, True, False, True)])
def test_conv1d_exact_cin8_vs_fp64(dil, res, acc, ragged):
    B, T, Cin, N, k = 3, 3000, 8, 8, 11
    pad = (k - 1) * dil // 2
    x, w = rnd(B, T, Cin, seed=41, scale=2.0), rnd(k, Cin, N, seed=42, scale=(k * Cin) ** -0.5)
    bias, r, y0 = rnd(N, seed=43, scale=0.1), rnd(B, T, N, seed=44), rnd(B, T, N, seed=45)
    lens = (3000, 1, 1234) if ragged else None
    y = y0.to(DEV).clone() if acc else torch.full((B, T, N), NAN, device=DEV)
    ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), dilation=dil, pad_left=pad, in_act=L.ACT_LRELU, in_slope=0.1, out_act=L.ACT_LRELU,
               out_slope=0.1, res=r.to(DEV) if res else None, alpha=0.5, out=y, accumulate=acc, backend=L.CONV_SIMT,
               x_lens=None if lens is None else torch.tensor(lens, dtype=torch.int32, device=DEV))
    torch.cuda.synchronize()
    got = y.cpu().double()
    for b in range(B):
        n = T if lens is None else lens[b]
        want = E.conv1d(x[b:b + 1, :n].double(), w.double(), bias.double(), dil, pad, E.ACT_LRELU, 0.1, E.ACT_LRELU, 0.1,
                        r[b:b + 1, :n].double() if res else None, 0.5, y0[b:b + 1, :n].double() if acc else None)
        assert (got[b:b + 1, :n] - want).abs().max().item() < 5e-6, b
