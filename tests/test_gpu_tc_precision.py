"""GPU: the tensor-core convolutions against fp64 across the operand magnitudes their splits represent (tests/tc_cases.py), with the
two per-element bars of tests/emul_cabi.py::tc_errors: (a) against the rounded-operand contract within E.TC_ACC_C 2^-24 S,
(b) against the unrounded fp64 conv within that plus R, the format's stated precision.  Also the shipped HiFi-GAN checkpoints' own layers on
the golden mels."""
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200 import ops, packing
from tests import emul_cabi as E
from tests import tc_cases as TC

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def tc_run(c, fmt, seg=False):
    """fs2_conv1d of a tc_cases layer on the tensor cores (backend 2) in format fmt; seg: the K-segmented tiles."""
    dv = lambda t: None if t is None else t.to(DEV)
    w = c["w"]
    if seg:
        wt, variant = packing.pack_conv_tc_segments(w), 2 | 4
    else:
        wt, variant = packing.pack_conv_tc(w, f8=fmt == "f8"), int(fmt == "f8")
    y = ops.conv1d(dv(c["x"]), dv(w), dv(c["bias"]), dilation=c["dil"], pad_left=c["pad"], in_act=c["in_act"], in_slope=0.1,
                   out_act=c["out_act"], out_slope=0.1, res=dv(c["res"]), alpha=c["alpha"],
                   out=None if c["y0"] is None else c["y0"].to(DEV).clone(), accumulate=c["y0"] is not None, row_lens=dv(c["lens"]),
                   w_tc=wt.to(DEV), backend=2, tc_variant=variant)
    torch.cuda.synchronize()
    return y.cpu()


def check(name, c, fmt, parity_log, utts=None, seg=False, **log):
    got = tc_run(c, fmt, seg)
    y_c, y64, S, R = TC.contract(c, fmt, utts, seg_cin=packing.SEG_CIN if seg else None)
    ea, eb = E.tc_errors(got if utts is None else got[utts], y_c, y64, S, R)
    bar = E.TC_SEG_ACC_C if seg else E.TC_ACC_C
    parity_log(name, fmt=fmt, err_contract=ea, err_fp64=eb, bar=bar, **log)
    assert ea <= bar and eb <= bar, (ea, eb)


MAG_PARAMS = [(v, "split3", n) for v in TC.MAG_VARIANTS for n in TC.SPLIT3_NS] + [(v, "f8", n) for v in TC.MAG_VARIANTS for n in TC.F8_NS]


@pytest.mark.parametrize("variant,fmt,N", MAG_PARAMS)
def test_conv_tc_magnitudes(variant, fmt, N, parity_log):
    """Every magnitude case at every work-item width of both formats."""
    check("test_conv_tc_magnitudes", TC.mag_case(variant, N), fmt, parity_log, case=variant, N=N)


@pytest.mark.parametrize("variant,fmt,N", TC.MAG_PERSISTENT)
def test_conv_tc_magnitudes_persistent(variant, fmt, N, parity_log):
    """Several work items per CTA, ragged lengths; the first and the last utterance against fp64."""
    c = TC.mag_case(variant, N, TC.MAG_PERSISTENT_SHAPE, TC.MAG_PERSISTENT_LENS)
    check("test_conv_tc_magnitudes_persistent", c, fmt, parity_log, utts=[0, 2], case=variant, N=N)


@pytest.mark.parametrize("case", TC.SEG_MAG_CASES, ids=[c[0] for c in TC.SEG_MAG_CASES])
def test_conv_tc_segmented_magnitudes(case, parity_log):
    """The K-segmented path with slices whose scales differ by powers of two: each slice must be scaled back with its own header."""
    check("test_conv_tc_segmented_magnitudes", TC.seg_case(case), "split3", parity_log, seg=True, case=case[0])


@pytest.mark.parametrize("fmt", ["split3", "f8"])
@pytest.mark.parametrize("xspec", [("scale", -12), ("chan", -14, 4), ("band", 256.0, 448.0)], ids=["x2^-12", "chan", "x[256,448)"])
def test_conv_tc_transpose_phase_group_magnitudes(fmt, xspec, parity_log):
    """One ConvTranspose phase group (u = 8, 2 taps, leaky_relu in) writing into the interleaved [B, T, u * C_out] rows."""
    u, cin, cout, T = 8, 128, 64, 700
    w = torch.randn(cin, cout, 2 * u, generator=torch.Generator().manual_seed(7)) * 0.05
    wa, _ = packing.split_conv_transpose(w, u)
    x = TC.make_x(xspec, 2, T, cin, seed=8)
    bias = (torch.randn(cout, generator=torch.Generator().manual_seed(9)) * 0.01 * float(x.abs().mean())).repeat(u // 2)
    out = torch.full((2, T, u * cout), float("nan"), device=DEV)
    ops.conv1d(x.to(DEV), wa.to(DEV), bias.to(DEV), pad_left=1, in_act=E.ACT_LRELU, in_slope=0.1, out=out[:, :, : u // 2 * cout],
               w_tc=packing.pack_conv_tc(wa, f8=fmt == "f8").to(DEV), backend=2, tc_variant=int(fmt == "f8"))
    torch.cuda.synchronize()
    y_c, y64, S, R = E.tc_contract(x, wa, bias, fmt, 1, 1, E.ACT_LRELU, 0.1)
    ea, eb = E.tc_errors(out.cpu()[:, :, : u // 2 * cout], y_c, y64, S, R)
    assert torch.isnan(out[:, :, u // 2 * cout:]).all()          # the other phase group's columns are not touched
    parity_log("test_conv_tc_transpose_phase_group_magnitudes", fmt=fmt, case=str(xspec), err_contract=ea, err_fp64=eb, bar=E.TC_ACC_C)
    assert ea <= E.TC_ACC_C and eb <= E.TC_ACC_C, (ea, eb)


# fs2_resstack: per-element bars with S and R summed over the group's layers (E.resstack_contract; empirical scales, not derived bounds).  Level (a) is against the same group
# built from per-layer fs2_conv1d calls on the same tiles, which compute the same rounded-operand products up to accumulation order
# (and, through it, rare roundings of an intermediate's split): RESSTACK_UNFUSED_C 2^-24 S.  Level (b) against fp64: RESSTACK_C 2^-24 S + R.
# Measured on an H100 80GB HBM3 at a 700 W power limit over test_resstack_fused, test_resstack_magnitudes and the shipped checkpoints'
# fused stages: 1.65 against the unfused group (universal, stage 3), and against fp64 every element within R itself (normalised excess 0).
RESSTACK_C = 1.0
RESSTACK_UNFUSED_C = 7.0


def resstack_check(name, x, kernels, dils, w1, b1, w2, b2, parity_log, **log):
    dv = lambda ws: [[t.to(DEV) for t in row] for row in ws]
    tiles = lambda ws: [[packing.pack_conv_tc(t, f8=True).to(DEV) for t in row] for row in ws]
    t1, t2 = tiles(w1), tiles(w2)
    got = ops.resstack(x.to(DEV), kernels, dils, t1, dv(b1), t2, dv(b2))

    def conv(x_, wt, b_, dil, pad, in_act=0, in_slope=0.0, out_act=0, out_slope=0.0, res=None, alpha=1.0, y_prev=None):
        return ops.conv1d(x_, wt[0], b_, dilation=dil, pad_left=pad, in_act=in_act, in_slope=in_slope, out_act=out_act, out_slope=out_slope,
                          res=res, alpha=alpha, out=y_prev, accumulate=y_prev is not None, w_tc=wt[1], backend=2, tc_variant=1)
    pair = lambda ws, ts: [list(zip(a, b)) for a, b in zip(dv(ws), ts)]
    unfused = E.resblock_group(x.to(DEV), kernels, dils, pair(w1, t1), dv(b1), pair(w2, t2), dv(b2), conv=conv)
    torch.cuda.synchronize()
    y64, S, R = E.resstack_contract(x, kernels, dils, w1, b1, w2, b2)
    _, eb = E.tc_errors(got.cpu(), y64, y64, S, R)
    eu, _ = E.tc_errors(got.cpu(), unfused.cpu().double(), y64, S, R)
    eb_unfused = E.tc_errors(unfused.cpu(), y64, y64, S, R)[1]
    parity_log(name, err_fp64=eb, bar=RESSTACK_C, err_vs_unfused=eu, bar_vs_unfused=RESSTACK_UNFUSED_C, err_unfused_fp64=eb_unfused, **log)
    assert torch.isfinite(got).all()
    assert eb <= RESSTACK_C and eu <= RESSTACK_UNFUSED_C, (eb, eu)


@pytest.mark.parametrize("C,N", [(32, 900), (64, 700)])
@pytest.mark.parametrize("xspec", [("scale", -12), ("scale", -6), ("scale", 0), ("scale", 6), ("chan", -14, 4)],
                         ids=["x2^-12", "x2^-6", "x1", "x2^6", "chan"])
def test_resstack_magnitudes(C, N, xspec, parity_log):
    """The fused ResBlock group at both channel counts, activation scale spanning 2^-12 .. 2^6 (weights and biases scale with it so that
    every layer's input stays in the band)."""
    kernels, dils = (3, 7, 11), ((1, 3, 5),) * 3
    x = TC.make_x(xspec, 2, N, C, seed=21)
    m = float(x.abs().mean())
    g = lambda s: torch.Generator().manual_seed(s)
    w1 = [[packing.conv_w(torch.randn(C, C, k, generator=g(100 + 10 * j + d)) * 0.6 * (C * k) ** -0.5) for d in range(3)] for j, k in enumerate(kernels)]
    w2 = [[packing.conv_w(torch.randn(C, C, k, generator=g(200 + 10 * j + d)) * 0.6 * (C * k) ** -0.5) for d in range(3)] for j, k in enumerate(kernels)]
    b1 = [[torch.randn(C, generator=g(300 + 10 * j + d)) * 0.05 * m for d in range(3)] for j in range(3)]
    b2 = [[torch.randn(C, generator=g(400 + 10 * j + d)) * 0.05 * m for d in range(3)] for j in range(3)]
    resstack_check("test_resstack_magnitudes", x, kernels, dils, w1, b1, w2, b2, parity_log, C=C, case=str(xspec))


# ------------------------------------------------------------------ shipped checkpoints
@pytest.mark.parametrize("name", ["LJSpeech", "universal"])
def test_real_checkpoint_layers(name, parity_log):
    """Every tensor-core layer of the shipped generator, alone, on its fp64 input from the golden mel (first utterance), in the format
    and fusion the default Generator hands the C ABI (Generator.effective_masks): per-layer convs through fs2_conv1d, the fused
    ResBlock groups through fs2_resstack."""
    from oracle import real_ckpt
    sd = real_ckpt.load(name)
    if sd is None:
        pytest.skip("real checkpoint fixture not present (run __graft_entry__.build() where the reference tree exists)")
    mel = torch.from_numpy(np.load(os.path.join(GOLD, f"hifigan_real_{name}.npz"))["mel"])[:1]
    convs, groups = TC.real_layers(*TC.hifigan_layer_inputs(sd, mel), TC.default_vocoder_masks())
    errs = {}
    for key, c, fmt in convs:
        y_c, y64, S, R = TC.contract(c, fmt)
        errs[key] = E.tc_errors(tc_run(c, fmt), y_c, y64, S, R)
        parity_log("test_real_checkpoint_layers", ckpt=name, layer=key, fmt=fmt, err_contract=errs[key][0], err_fp64=errs[key][1],
                   bar=E.TC_ACC_C)
    for stage, x, w1, b1, w2, b2 in groups:
        resstack_check("test_real_checkpoint_layers_resstack", x, (3, 7, 11), ((1, 3, 5),) * 3, w1, b1, w2, b2, parity_log, ckpt=name,
                       stage=stage)
    bad = {k: v for k, v in errs.items() if max(v) > E.TC_ACC_C}
    assert not bad, bad
