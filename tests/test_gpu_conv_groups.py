"""GPU: the tensor-core conv's channel-block groups (fs2_conv_tc_plan_t::NG) at every group shape of tests/conv_group_cases.py.

Each case runs at the batch where the device's own plan (its SM count, not 132) picks the case's NG, into an output poisoned with NaN
around the written columns, and is checked three ways:
  1. bit for bit against the same conv computed one channel block per launch (N = NB: one block, NG = 1), every launch reading its
     block's tiles from the SAME packed buffer, header included, so that both sides multiply the same operand bits;
  2. per element against fp64 on the first and the last utterance (every group's blocks appear in both: items are ordered
     (group, utterance, tile)), with the two bars of tests/emul_cabi.py::tc_errors, plus tanhf's 2 ulp where the epilogue is tanh;
  3. the NaN sentinels outside the written columns untouched.
The windowed and multi-generator entry points are checked through Generator at batches where the layer named plans NG >= 2 on the
device: the V2 offline forward (ups 0 phase groups), a V1 stream pool (conv_pre) and a pool of two generators whose weight-scale
headers and biases differ in every layer."""
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, ops, packing, synth
from oracle import fs2_oracle as O
from tests import conv_group_cases as G
from tests import emul_cabi as E
from tests import tc_cases as TC
from tests.test_gpu_hifigan_v2 import WAV_TOL, _generator as _v2_generator
from tests.test_gpu_stream_multi import _run
from tests.test_gpu_stream_vocoder import _generator

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN = float("nan")


def device_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def block_tiles(wt, k, taps, cin, nb):
    """The packed weights of channel block k alone (a buffer for N = nb): wt's 128-byte header, then block k's tiles, which
    packing.pack_conv_tc stores [N / NB][Cin / 16][taps][2 planes][2 K-chunks][NB][16 bytes]."""
    per = (cin // 16) * taps * 64 * nb
    hdr = packing.TC_HEADER_BYTES
    return torch.cat([wt[:hdr], wt[hdr + k * per:hdr + (k + 1) * per]])


def ulp32(v):
    a = v.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))) - a).double()


def errors(got, y_c, y64, S, R, slack):
    """tc_errors' two normalised errors, with `slack` (per element) allowed on top of both bars: tanhf's 2 ulp."""
    def norm(d):
        d = (d - slack).clamp_min(0.0)
        r = torch.where(S > 0, d / (E.U24 * S.clamp_min(1e-300)), torch.where(d > 0, float("inf"), 0.0))
        return torch.nan_to_num(r, nan=float("inf")).max().item()
    g = got.double()
    return norm((g - y_c).abs()), norm(((g - y64).abs() - R).clamp_min(0.0))


def _inputs(c, B, seed):
    """Host tensors of case c at batch B: x, w, bias, res, y0 (None where the case has none) and the lengths (a list or None)."""
    T, Cin, N, taps = c["T"], c["Cin"], c["N"], c["taps"]
    g = lambda s: torch.Generator().manual_seed(seed + s)
    x = TC.make_x(c["x"], B, T, Cin, seed=seed)
    w = TC.make_w(("rms", 0), taps, Cin, N, seed=seed + 2)
    mag = float(x.abs().mean()) * float(w.abs().mean()) * (taps * Cin) ** 0.5
    bias = torch.randn(N, generator=g(3)) * 0.1 * mag if c["bias"] else None
    res = torch.randn(B, T, N, generator=g(4)) * mag if c["res"] else None
    y0 = torch.randn(B, T, N, generator=g(5)) * mag if c["acc"] else None
    lens = G.lens_of(c, B) if c["lens"] else None
    return x, w, bias, res, y0, lens


def _x_on_device(c, x, lens):
    """x as the kernel reads it: a column slice of wider rows (x_cols) with NaN in every column, row and batch gap it must not read,
    and NaN in the rows at or past a ragged utterance's length (read as zero)."""
    B, T, Cin = x.shape
    xt, xo = c["x_cols"] or (Cin, 0)
    extra = 5 if c["x_cols"] else 0
    buf = torch.full((B, T + extra, xt), NAN, device=DEV)
    view = buf[:, :T, xo:xo + Cin]
    view.copy_(x.to(DEV))
    if c["lens"] == "x_lens":
        for b, n in enumerate(lens):
            view[b, n:] = NAN
    return view


def _out(c, B, y0):
    """The output: NaN rows of y_cols[0] floats (or N), the written columns a view of them, holding y0 when accumulating."""
    T, N = c["T"], c["N"]
    yt, yo = c["y_cols"] or (N, 0)
    buf = torch.full((B, T, yt), NAN, device=DEV)
    view = buf[:, :, yo:yo + N]
    if y0 is not None:
        view.copy_(y0.to(DEV))
    return buf, view


def _conv(c, x, w, bias, res, out, wt, lens_d):
    ops.conv1d(x, w, bias, dilation=c["dil"], pad_left=c["pad"], in_act=c["in_act"], in_slope=0.1, out_act=c["out_act"], out_slope=0.1,
               res=res, alpha=c["alpha"], out=out, accumulate=c["acc"], w_tc=wt, backend=L.CONV_TC, tc_variant=G.FMT_VARIANT[c["fmt"]],
               row_lens=lens_d if c["lens"] == "row_lens" else None, x_lens=lens_d if c["lens"] == "x_lens" else None)


def _live(c, B, lens):
    """[B, T, 1] bool: the rows whose values are specified (below each utterance's length under x_lens, every row otherwise)."""
    t = torch.arange(c["T"], device=DEV)[None, :, None]
    if c["lens"] != "x_lens":
        return torch.ones(B, c["T"], 1, dtype=torch.bool, device=DEV)
    return t < torch.tensor(lens, device=DEV)[:, None, None]


@pytest.mark.parametrize("c", G.CASES, ids=[c["name"] for c in G.CASES])
def test_grouped_conv_equals_one_block_per_launch_and_fp64(c, parity_log):
    sms = device_sms()
    B = G.choose_batch(c, sms)
    p = G.plan(c, B, sms)
    NB, N, T = p["NB"], c["N"], c["T"]
    nblk = N // NB
    assert p["NG"] == c["NG"] and nblk > 1, p
    assert G.plan(dict(c, N=NB, y_cols=None), B, sms)["NG"] == 1
    x, w, bias, res, y0, lens = _inputs(c, B, seed=len(c["name"]) * 31 + c["NG"])
    wt = packing.pack_conv_tc(w, f8=c["fmt"] == "f8").to(DEV)
    xd, wd = _x_on_device(c, x, lens), w.to(DEV)
    bd = None if bias is None else bias.to(DEV)
    rd = None if res is None else res.to(DEV)
    lens_d = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=DEV)

    got_buf, got = _out(c, B, y0)
    _conv(c, xd, wd, bd, rd, got, wt, lens_d)
    ref_buf, ref = _out(c, B, y0)
    for k in range(nblk):
        s = slice(k * NB, (k + 1) * NB)
        _conv(c, xd, wd[:, :, s].contiguous(), None if bd is None else bd[s], None if rd is None else rd[:, :, s], ref[:, :, s],
              block_tiles(wt, k, c["taps"], c["Cin"], NB), lens_d)
    torch.cuda.synchronize()

    # 1. the grouped launch against one block per launch, on every specified row
    live = _live(c, B, lens).expand(B, T, N)
    assert torch.equal(got[live], ref[live])
    assert not torch.isnan(got[live]).any()
    # 3. the sentinels around the written columns
    yo = (c["y_cols"] or (N, 0))[1]
    assert torch.isnan(got_buf[:, :, :yo]).all() and torch.isnan(got_buf[:, :, yo + N:]).all()
    # 2. fp64 on the first and the last utterance (ragged: each alone on its own rows, and the 1-row one too)
    tanh = c["out_act"] == L.ACT_TANH
    utts = [0, B - 1] + ([2] if c["lens"] == "x_lens" and B > 3 else [])
    worst = [0.0, 0.0]
    for b in utts:
        n = lens[b] if c["lens"] == "x_lens" else T
        sel = lambda t: None if t is None else t[b:b + 1, :n]
        rl = torch.tensor([lens[b]]) if c["lens"] == "row_lens" else None
        y_c, y64, S, R = E.tc_contract(sel(x), w, bias, c["fmt"], c["dil"], c["pad"], c["in_act"], 0.1, c["out_act"], 0.1, sel(res),
                                       c["alpha"], sel(y0), rl)
        e = errors(got[b:b + 1, :n].cpu(), y_c, y64, S, R, 2 * ulp32(y_c) if tanh else 0.0)
        worst = [max(worst[0], e[0]), max(worst[1], e[1])]
    parity_log("test_grouped_conv_equals_one_block_per_launch_and_fp64", case=c["name"], cls=sorted(G.classes(c)), fmt=c["fmt"],
               NB=NB, NG=p["NG"], B=B, sms=sms, err_contract=worst[0], err_fp64=worst[1], bar=E.TC_ACC_C,
               frac=max(worst) / E.TC_ACC_C)
    assert worst[0] <= E.TC_ACC_C and worst[1] <= E.TC_ACC_C, worst


# ------------------------------------------------------------------ the vocoder's entry points with more blocks than NG
def _launch(m, T, f0, f1, layer, stage=-1):
    return next(l for l in L.vocoder_window_plan(m, T, f0, f1) if l.layer == layer and l.stage == stage)


def _layer_case(m, layer, stage, rows):
    """conv_group_cases.case of a vocoder launch: conv_pre, or a ConvTranspose phase group, at `rows` rows per utterance."""
    if layer == L.VW_CONV_PRE:
        return G.case("conv_pre", (), "f8" if m.f8_mask & 1 else "split3", 80, m.c0, 7, 0, T=rows)
    u, C = m.rates[stage], m.c0 >> stage
    return G.case(f"ups.{stage}", (), "f8" if m.f8_mask & (2 << stage) else "split3", C, u // 2 * (C // 2), 2, 0, pad=1,
                  in_act=L.ACT_LRELU, y_cols=(u * (C // 2), 0), T=rows)


@pytest.mark.parametrize("ragged", [False, True])
def test_v2_offline_batch_with_groups_equals_each_utterance_alone(ragged):
    """HiFi-GAN V2 offline at a batch where its ups 0 phase groups (128 -> 4 x 64, 4 blocks of 64) plan NG >= 2 on the device:
    every utterance bit for bit equal to itself alone (one utterance: NG = 1), the first and the last within WAV_TOL of the oracle."""
    gen, sd = _v2_generator(13)
    frames = 300
    gen(synth.make_mel(1, 4, seed=1).to(DEV))          # packs the weights
    m = gen._packed[0]
    up0 = _launch(m, frames, 0, frames, L.VW_UP_A, 0)
    c = _layer_case(m, L.VW_UP_A, 0, up0.y1 - up0.y0)
    B = G.choose_batch(dict(c, NG=2), device_sms())
    assert up0.y1 - up0.y0 == frames and G.plan(c, B, device_sms())["NG"] >= 2
    assert G.plan(c, 1, device_sms())["NG"] == 1
    mel = synth.make_mel(B, frames, seed=17)
    lens = None
    if ragged:
        lens = [frames, 0, 1] + [(b * 97 + 11) % (frames + 1) for b in range(3, B - 1)] + [frames - 29]
    wav = gen(mel.to(DEV), None if lens is None else torch.tensor(lens))
    torch.cuda.synchronize()
    up = 256
    for b in range(B):
        n = frames if lens is None else lens[b]
        if n == 0:
            assert torch.equal(wav[b], torch.zeros_like(wav[b])), b
            continue
        alone = gen(mel[b:b + 1, :, :n].to(DEV))[0]
        assert torch.equal(wav[b, :, :up * n], alone), (b, n)
        assert torch.equal(wav[b, :, up * n:], torch.zeros_like(wav[b, :, up * n:])), (b, n)
        if b in (0, B - 1):
            assert (alone.cpu() - O.hifigan_forward(sd, mel[b:b + 1, :, :n])[0]).abs().max().item() < WAV_TOL, b


def test_v1_stream_pool_with_grouped_conv_pre_equals_each_forward():
    """512 V1 streams in one pool, 32-frame chunks: conv_pre (80 -> 512, 4 blocks) plans NG >= 2 on the window's rows.  Each stream's
    chunks, joined, equal its own forward."""
    gen = _generator(configs.HIFIGAN_CONFIG, seed=7)
    n, chunk = 512, 32
    pool = gen.stream_pool(chunk_frames=chunk)
    m = (gen._packed or gen._pack())[0]
    pre = _launch(m, 1 << 20, 1 << 16, (1 << 16) + chunk, L.VW_CONV_PRE)
    assert G.plan(_layer_case(m, L.VW_CONV_PRE, -1, pre.y1 - pre.y0), n, device_sms())["NG"] >= 2
    mels = [synth.make_mel(1, 33 + (k * 37) % 64, seed=300 + k)[0].to(DEV) for k in range(n)]
    out = _run(pool, mels, [0] * n, [0] * n)
    for k, mel in enumerate(mels):
        assert torch.equal(out[k], gen(mel[None])), k


def _rescaled(gen, seed):
    """gen's architecture with every tensor-core layer's weights times 2^3 or 2^-3 (the two convs of a ResBlock pair and successive
    stages alternate, so the signal stays in range) and other biases: every weight-scale header and bias differs from gen's."""
    g = torch.Generator().manual_seed(seed)
    out = _generator(configs.HIFIGAN_CONFIG, seed=3)
    with torch.no_grad():
        for name, prm in out.named_parameters():
            if name.startswith("conv_post"):
                continue
            if name.endswith("weight"):
                up = name.startswith("ups.") and int(name.split(".")[1]) % 2 == 0 or ".convs1." in name
                prm.mul_(8.0 if up else 0.125)
            elif name.endswith("bias"):
                prm.add_((torch.randn(prm.shape, generator=g) * 0.05).to(prm.device))
    out._invalidate()
    return out


def test_multi_generator_pool_reads_each_units_own_header_and_bias():
    """Two generators with the same architecture whose every tensor-core layer's weight-scale header (a power of two: 2^3 apart) and
    bias differ, 96 streams in one pool, the 128-channel stage planned at NG >= 2: each stream equals its own generator's forward."""
    gens = [_generator(configs.HIFIGAN_CONFIG, seed=3)]
    gens.append(_rescaled(gens[0], seed=29))
    n, chunk = 96, 32
    pool = gens[0].stream_pool(chunk_frames=chunk, generators=gens[1:])
    m = (gens[0]._packed or gens[0]._pack())[0]
    rb = _launch(m, 1 << 20, 1 << 16, (1 << 16) + chunk, L.VW_RB_CONV1, 1)
    assert G.plan(G.case("rb", (), "f8", 128, 128, 3, 0, T=rb.y1 - rb.y0), n, device_sms())["NG"] >= 2
    pk = [(g._packed or g._pack())[1] for g in gens]
    hdr = lambda t: abs(float(t[:4].cpu().view(torch.float32)))
    tiles = [k for k in pk[0] if k.endswith("_tc")]
    assert tiles and all(hdr(pk[1][k]) in (8 * hdr(pk[0][k]), hdr(pk[0][k]) / 8) for k in tiles if not k.startswith("w_post"))
    biases = [k for k in pk[0] if k == "b_pre" or k.endswith((".b", ".b1", ".b2"))]
    assert biases and all(not torch.equal(pk[0][k], pk[1][k]) for k in biases)
    mels = [synth.make_mel(1, 40 + (k * 13) % 57, seed=500 + k)[0].to(DEV) for k in range(n)]
    which = [(k * 5) % 2 for k in range(n)]
    out = _run(pool, mels, which, [int(k % 7 == 0) for k in range(n)])
    for k, mel in enumerate(mels):
        assert torch.equal(out[k], gens[which[k]](mel[None])), (k, which[k])
