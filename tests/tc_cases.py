"""Magnitude cases for the tensor-core convolutions (TEST INFRASTRUCTURE, shared by tests/test_tc_precision_cpu.py and
tests/test_gpu_tc_precision.py).

The operand splits of the tensor-core kernels lose precision in magnitude bands that N(0, 1) activations and (taps Cin)^-1/2 weights
never reach: below about 2^-3 the fp16 lo plane is subnormal (an absolute floor of 2^-25 per operand), from 256 on the E4M3
correction's lo * 2^12 saturates, beyond 448 its hi does too, and a weight far below its layer's maximum (the header scale) has a
subnormal lo.  Every case here puts one layer's operands into one of those bands, or mixes them inside one layer.
"""
import torch

from tests import emul_cabi as E


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _signed_band(shape, lo, hi, seed):
    """Magnitudes uniform in [lo, hi), random signs."""
    m = lo + (hi - lo) * torch.rand(*shape, generator=_g(seed), dtype=torch.float64)
    s = torch.where(torch.rand(*shape, generator=_g(seed + 1)) < 0.5, -1.0, 1.0)
    return (m * s).float()


# Activations.  ("scale", e): N(0, 1) * 2^e for the whole layer; ("band", lo, hi): |x| uniform in [lo, hi); ("chan", e0, e1): N(0, 1)
# times a per-channel 2^u, u uniform in [e0, e1]; ("cancel",): channel pairs x[2i + 1] = x[2i].
# Weights.  ("rms", e): N(0, 1) (taps Cin)^-1/2 2^e; ("max", e): the same rescaled so that max|w| = 2^e (the header scale then
# spans 2^-20 .. 2^10 of the table); ("outliers", f): one weight in 64 is f times the rms, so most weights sit far below the layer
# maximum; ("cancel",): w[2i + 1] = -w[2i] (1 + 2^-10 r), so y ~ 2^-10 S; ("segments", e...): K-segment k (tap-major, 256 input
# channels each) scaled by 2^e[k % len(e)].
MAG_VARIANTS = {
    "x2^-12": dict(x=("scale", -12)),
    "x2^-6": dict(x=("scale", -6)),
    "x1": dict(x=("scale", 0)),
    "x2^6": dict(x=("scale", 6)),
    "x[224,256)": dict(x=("band", 224.0, 256.0)),
    "x[256,448)": dict(x=("band", 256.0, 448.0)),
    "x[448,4096)": dict(x=("band", 448.0, 4096.0)),
    "x[2^14,65504]": dict(x=("band", 16384.0, 65504.0)),
    "x_chan2^-14..2^4": dict(x=("chan", -14, 4)),
    "w_max2^-20": dict(w=("max", -20)),
    "w_max2^10": dict(w=("max", 10)),
    "w_outliers": dict(x=("scale", -4), w=("outliers", 1e3)),
    "cancel": dict(x=("cancel",), w=("cancel",)),
    # the epilogue terms (lrelu in and out, residual, alpha, accumulate) around small operands
    "x2^-12_epilogue": dict(x=("scale", -12), act=(E.ACT_LRELU, E.ACT_LRELU), res=True, alpha=1.0 / 3, acc=True),
}

# The base layer of the table: B, T, Cin, taps, dilation, pad_left
MAG_SHAPE = (2, 260, 32, 3, 1, 1)
# The output widths: every work-item width NB the dispatcher instantiates (N <= 128: NB = N for split3; N <= 64 for f8), and
# N = 192, two or three NB blocks (96 / 64)
SPLIT3_NS = (16, 32, 48, 64, 80, 96, 112, 128, 192)
F8_NS = (16, 32, 48, 64, 192)
# Several work items per CTA on 132 SMs (3 x 24000 rows = 564 items per channel block), ragged lengths: (variant, fmt, N)
MAG_PERSISTENT = [("x2^-12", "split3", 64), ("x_chan2^-14..2^4", "f8", 48), ("w_outliers", "split3", 128), ("x[256,448)", "f8", 64),
                  ("x2^-12_epilogue", "f8", 32), ("cancel", "split3", 96)]
MAG_PERSISTENT_SHAPE = (3, 24000, 16, 3, 1, 1)
MAG_PERSISTENT_LENS = (24000, 13001, 23873)


def make_x(spec, B, T, Cin, seed=1):
    kind = spec[0]
    if kind == "scale":
        return torch.randn(B, T, Cin, generator=_g(seed)) * 2.0 ** spec[1]
    if kind == "band":
        return _signed_band((B, T, Cin), spec[1], spec[2], seed)
    if kind == "chan":
        u = spec[1] + (spec[2] - spec[1]) * torch.rand(Cin, generator=_g(seed + 7))
        return torch.randn(B, T, Cin, generator=_g(seed)) * torch.exp2(u)
    if kind == "cancel":
        return torch.randn(B, T, Cin // 2, generator=_g(seed)).repeat_interleave(2, dim=2)
    raise ValueError(spec)


def make_w(spec, taps, Cin, N, seed=2):
    w = torch.randn(taps, Cin, N, generator=_g(seed)) * (taps * Cin) ** -0.5
    kind = spec[0]
    if kind == "rms":
        return w * 2.0 ** spec[1]
    if kind == "max":
        return (w / w.abs().max() * 2.0 ** spec[1]).float()
    if kind == "outliers":
        pick = torch.rand(taps, Cin, N, generator=_g(seed + 3)) < 1.0 / 64
        return torch.where(pick, w * spec[1], w)
    if kind == "cancel":
        r = torch.rand(taps, Cin // 2, N, generator=_g(seed + 5)) * 2.0 - 1.0
        w0 = w[:, 0::2]
        return torch.stack([w0, -w0 * (1 + r * 2.0 ** -10)], dim=2).reshape(taps, Cin, N)
    if kind == "segments":
        f = torch.tensor([2.0 ** e for e in spec[1:]])
        nk = Cin // 256
        seg = torch.arange(taps * nk).reshape(taps, nk) % len(f)
        return w * f[seg].repeat_interleave(256, dim=1)[..., None]
    raise ValueError(spec)


def mag_case(variant, N, shape=MAG_SHAPE, lens=None):
    """A layer of the table: dict(x, w, bias, res, y0, lens, dil, pad, in_act, out_act, alpha).  The bias, residual and accumulated output
    scale with the products so that they do not swamp them."""
    v = MAG_VARIANTS[variant]
    B, T, Cin, taps, dil, pad = shape
    x = make_x(v.get("x", ("scale", 0)), B, T, Cin)
    w = make_w(v.get("w", ("rms", 0)), taps, Cin, N)
    mag = float(x.abs().mean()) * float(w.abs().mean()) * (taps * Cin) ** 0.5
    in_act, out_act = v.get("act", (E.ACT_NONE, E.ACT_NONE))
    c = dict(x=x, w=w, bias=torch.randn(N, generator=_g(3)) * 0.1 * mag, dil=dil, pad=pad, in_act=in_act, out_act=out_act,
             alpha=v.get("alpha", 1.0), res=None, y0=None, lens=None if lens is None else torch.tensor(lens, dtype=torch.int32))
    if v.get("res"):
        c["res"] = torch.randn(B, T, N, generator=_g(4)) * mag
    if v.get("acc"):
        c["y0"] = torch.randn(B, T, N, generator=_g(5)) * mag
    return c


def contract(c, fmt, utts=None, seg_cin=None):
    """E.tc_contract of a mag_case layer (in_slope = out_slope = 0.1) on the utterances utts (all when None)."""
    sel = (lambda t: t) if utts is None else (lambda t: None if t is None else t[utts])
    return E.tc_contract(sel(c["x"]), c["w"], c["bias"], fmt, c["dil"], c["pad"], c["in_act"], 0.1, c["out_act"], 0.1, sel(c["res"]),
                         c["alpha"], sel(c["y0"]), sel(c["lens"]), seg_cin=seg_cin)


# K-segmented encoder / predictor layers (FS2_TC_VARIANT_SEGMENTED: one scale per (tap, 256-channel) slice): (name, x spec, B, T, Cin,
# N, taps, pad, segment exponents).  Segment maxima that differ by powers of two, so that a kernel decoding one slice with another's
# header is off by that power.
SEG_MAG_CASES = [
    ("seg_w2^0,-3,5,-9_x1", ("scale", 0), 2, 200, 1024, 128, 1, 0, (0, -3, 5, -9)),
    ("seg_w2^4,-6_x2^-12", ("scale", -12), 2, 300, 512, 64, 3, 1, (4, -6, 0)),
    ("seg_w2^-2,2_chan", ("chan", -14, 4), 2, 150, 256, 192, 9, 4, (-2, 2, 0, 7, -11)),
    ("seg_w2^0,8_x2^6", ("scale", 6), 2, 260, 512, 256, 1, 0, (0, 8)),
]


def seg_case(case):
    name, xs, B, T, Cin, N, taps, pad, exps = case
    x = make_x(xs, B, T, Cin)
    w = make_w(("segments",) + tuple(exps), taps, Cin, N)
    mag = float(x.abs().mean()) * float(w.abs().mean()) * (taps * Cin) ** 0.5
    return dict(x=x, w=w, bias=torch.randn(N, generator=_g(3)) * 0.1 * mag, dil=1, pad=pad, in_act=E.ACT_NONE, out_act=E.ACT_NONE,
                alpha=1.0, res=None, y0=None, lens=None)


def hifigan_layer_inputs(sd, mel, stages=None):
    """The shipped generator in fp64 on mel [B, 80, T], channels-last inputs of every tensor-core layer: {"conv_pre": mel, "ups.i": x
    before its leaky_relu, "rb.i": the ResBlock group input of stage i, "rb.i.j.d.1" / "rb.i.j.d.2": the inputs of convs1.d / convs2.d
    of kernel size j before their leaky_relu}.  Also returns the folded fp64 state_dict."""
    import torch.nn.functional as F
    from oracle import fs2_oracle as O
    sd = {k: v.double() for k, v in O.fold_weight_norm(sd).items()}
    rates, ks, dils = (8, 8, 2, 2), (3, 7, 11), (1, 3, 5)
    cl = lambda t: t.transpose(1, 2).contiguous()
    out = {"conv_pre": cl(mel.double())}
    x = F.conv1d(mel.double(), sd["conv_pre.weight"], sd["conv_pre.bias"], padding=3)
    for i, u in enumerate(rates):
        if stages is not None and i > max(stages):
            break
        out[f"ups.{i}"] = cl(x)
        x = F.conv_transpose1d(F.leaky_relu(x, 0.1), sd[f"ups.{i}.weight"], sd[f"ups.{i}.bias"], stride=u, padding=u // 2)
        out[f"rb.{i}"] = cl(x)
        acc = 0
        for j, k in enumerate(ks):
            r = x
            p = f"resblocks.{i * len(ks) + j}"
            for m, d in enumerate(dils):
                out[f"rb.{i}.{j}.{m}.1"] = cl(r)
                t = F.conv1d(F.leaky_relu(r, 0.1), sd[f"{p}.convs1.{m}.weight"], sd[f"{p}.convs1.{m}.bias"], dilation=d, padding=(k * d - d) // 2)
                out[f"rb.{i}.{j}.{m}.2"] = cl(t)
                r = F.conv1d(F.leaky_relu(t, 0.1), sd[f"{p}.convs2.{m}.weight"], sd[f"{p}.convs2.{m}.bias"], padding=(k - 1) // 2) + r
            acc = acc + r
        x = acc / len(ks)
    return out, sd


def default_vocoder_masks():
    """(f8_mask, fused_mask, pair_mask, pair_kmax) the default Generator hands the C ABI (Generator.effective_masks, no GPU needed)."""
    from fastspeech2_b200 import configs
    from fastspeech2_b200.hifigan import AttrDict, Generator
    return Generator(AttrDict(configs.HIFIGAN_CONFIG)).effective_masks()


def real_layers(ins, f, masks):
    """The shipped generator's tensor-core work under the given effective masks, on the inputs of hifigan_layer_inputs: per-layer convs
    as (key, mag_case-style layer, fmt) and fused ResBlock groups as (stage, x, w1, b1, w2, b2).  A stage in pair_mask (a pair-fused
    stage) is not covered here, so it is refused."""
    from fastspeech2_b200 import packing
    f8_mask, fused_mask, pair_mask, _ = masks
    assert pair_mask == 0, "pair-fused ResBlock stages are not covered by this layer list"
    cw = lambda k: packing.conv_w(f[k + ".weight"]).float()
    fmt_of = lambda stage: "f8" if (f8_mask >> (stage + 1)) & 1 else "split3"
    lay = lambda x, w, b, dil=1, pad=0, in_act=E.ACT_NONE: dict(x=x.float(), w=w, bias=b.float(), dil=dil, pad=pad, in_act=in_act,
                                                               out_act=E.ACT_NONE, alpha=1.0, res=None, y0=None, lens=None)
    convs = [("conv_pre", lay(ins["conv_pre"], cw("conv_pre"), f["conv_pre.bias"], pad=3), fmt_of(-1))]
    groups = []
    for i, u in enumerate((8, 8, 2, 2)):
        wa, wb = packing.split_conv_transpose(f[f"ups.{i}.weight"].float(), u)
        bt = f[f"ups.{i}.bias"].float().repeat(u // 2)
        convs.append((f"ups.{i}.a", lay(ins[f"ups.{i}"], wa, bt, pad=1, in_act=E.ACT_LRELU), fmt_of(i)))
        convs.append((f"ups.{i}.b", lay(ins[f"ups.{i}"], wb, bt, pad=0, in_act=E.ACT_LRELU), fmt_of(i)))
        p = lambda j, m, n: f"resblocks.{i * 3 + j}.convs{n}.{m}"
        if (fused_mask >> i) & 1:
            groups.append((i, ins[f"rb.{i}"].float(), [[cw(p(j, m, 1)) for m in range(3)] for j in range(3)],
                           [[f[p(j, m, 1) + ".bias"].float() for m in range(3)] for j in range(3)],
                           [[cw(p(j, m, 2)) for m in range(3)] for j in range(3)],
                           [[f[p(j, m, 2) + ".bias"].float() for m in range(3)] for j in range(3)]))
            continue
        for j, k in enumerate((3, 7, 11)):
            for m, d in enumerate((1, 3, 5)):
                convs.append((p(j, m, 1), lay(ins[f"rb.{i}.{j}.{m}.1"], cw(p(j, m, 1)), f[p(j, m, 1) + ".bias"], d, (k - 1) * d // 2,
                                              E.ACT_LRELU), fmt_of(i)))
                convs.append((p(j, m, 2), lay(ins[f"rb.{i}.{j}.{m}.2"], cw(p(j, m, 2)), f[p(j, m, 2) + ".bias"], 1, (k - 1) // 2,
                                              E.ACT_LRELU), fmt_of(i)))
    return convs, groups
