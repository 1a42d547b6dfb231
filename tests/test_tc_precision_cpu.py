"""CPU: the tensor-core operand formats against their definitions, without a GPU.

  * the packer's tiles decode (tests/emul_cabi.py::unpack_conv_tc) to exactly the weight operands the emulator derives from the
    format definition, at every work-item width and in every K-segment, so that a layout or scale bug cannot hide in both;
  * the rounded-operand contract stays within R, the format's stated precision, over the whole magnitude table
    (tests/tc_cases.py), and R is not vacuous;
  * kernel faults, emulated in fp64, leave the level-(a) bar of the GPU tests by at least 10x on some case of the table;
  * the shipped HiFi-GAN checkpoints keep every activation of their f16 + f8 layers below 256, where the correction does not
    saturate.
"""
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200 import packing
from tests import emul_cabi as E
from tests import tc_cases as TC

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("fmt,N", [("split3", n) for n in TC.SPLIT3_NS] + [("f8", n) for n in TC.F8_NS])
@pytest.mark.parametrize("wspec", [("rms", 0), ("max", -20), ("max", 10), ("outliers", 1e3)])
def test_packed_tiles_decode_to_emulated_operands(fmt, N, wspec):
    """pack_conv_tc at the NB the dispatcher picks, decoded from its bytes alone, equals the emulator's weight operands bit for bit."""
    w = TC.make_w(wspec, 3, 48, N)
    nb = packing.conv_tc_block(N, 64 if fmt == "f8" else 128)
    buf = packing.pack_conv_tc(w, f8=fmt == "f8")
    assert buf is not None and int(buf[4]) == (fmt == "f8")
    for got, want in zip(E.unpack_conv_tc(buf, 3, 48, N, nb), E.w_planes(w, fmt)):
        assert torch.equal(got, want)


@pytest.mark.parametrize("case", TC.SEG_MAG_CASES, ids=[c[0] for c in TC.SEG_MAG_CASES])
def test_packed_segments_decode_to_emulated_operands(case):
    """pack_conv_tc_segments: every (tap, 256-channel) slice carries its own header, and decodes to the emulator's operands of that
    slice.  The table's slices differ in scale, so a slice decoded with another's header would not match."""
    _, _, _, _, Cin, N, taps, _, _ = case
    w = TC.seg_case(case)["w"]
    buf = packing.pack_conv_tc_segments(w)
    seg_bytes = 128 + 1024 * N
    want = E._segmented(lambda v: E.w_planes(v, "split3"), w, packing.SEG_CIN)
    scales = set()
    for t in range(taps):
        for k in range(Cin // packing.SEG_CIN):
            i = t * (Cin // packing.SEG_CIN) + k
            seg = buf[i * seg_bytes:(i + 1) * seg_bytes]
            scales.add(float(seg[:4].view(torch.float32)))
            got = E.unpack_conv_tc(seg, 1, packing.SEG_CIN, N, 64)
            for g_, w_ in zip(got, want):
                assert torch.equal(g_, w_[t:t + 1, k * packing.SEG_CIN:(k + 1) * packing.SEG_CIN])
    assert len(scales) > 1 or taps * Cin // packing.SEG_CIN == 1


def _variants(fmt):
    return [(v, fmt, N) for v in TC.MAG_VARIANTS for N in (64, 192)]


@pytest.mark.parametrize("variant,fmt,N", _variants("split3") + _variants("f8"))
def test_contract_within_stated_precision(variant, fmt, N):
    """|y_c - y64| <= R on every element: the rounded-operand contract is as accurate as the format says."""
    c = TC.mag_case(variant, N)
    y_c, y64, S, R = TC.contract(c, fmt)
    assert ((y_c - y64).abs() <= R).all(), ((y_c - y64).abs() / R).max().item()


# R is the sum of worst cases; the largest element of |y_c - y64| / R over the table must come within this factor of 1 in each format
# (measured: 0.93 split3, 0.56 f8), so that R is not a loose bound under which a lost bit could hide.
R_TIGHT = 0.25


@pytest.mark.parametrize("fmt", ["split3", "f8"])
def test_stated_precision_is_reached(fmt):
    worst = 0.0
    for variant in TC.MAG_VARIANTS:
        y_c, y64, S, R = TC.contract(TC.mag_case(variant, 64), fmt)
        worst = max(worst, ((y_c - y64).abs() / R.clamp_min(1e-300)).max().item())
    assert R_TIGHT <= worst <= 1.0, worst


def test_split3_floor_below_eighth():
    """The fp16 split keeps 22 significant bits only while the lo plane is normal: below |a| ~ 2^-3 the absolute floor 2^-25 takes
    over, and at |a| = 2^-12 the relative representation error is about 2^-13 instead of 2^-23."""
    a = torch.tensor([1.0 + 2.0 ** -20, 2.0 ** -12 * (1 + 2.0 ** -13 + 2.0 ** -20)]).float()
    hi, lo, _ = E.a_planes(a, "split3")
    rel = ((hi + lo - a.double()).abs() / a.double()).tolist()
    assert rel[0] < 2.0 ** -22 and rel[1] > 2.0 ** -16


# ------------------------------------------------------------------ fault emulations
# Each fault changes the operands one kernel would multiply; its contract must leave the level-(a) bar (E.TC_ACC_C 2^-24 S) by at
# least FAULT_FACTOR on some case of the table (FAULTS), or on every shape a test runs (test_dropped_terms_exceed_bar_*).
FAULT_FACTOR = 10.0


def _fault_contract(c, fmt, fault, seg_cin=None):
    a = E.act_operand(c["x"], c["in_act"], 0.1)
    A = E.a_planes(a, fmt)
    W = E._segmented(lambda v: E.w_planes(v, fmt), c["w"], seg_cin)
    if fault == "lo_flush":                          # split_f16x2 flushing a subnormal lo to zero
        A[1] = torch.where(A[1].abs() < 2.0 ** -14, 0.0, A[1])
    elif fault == "f8_lo_2^11":                      # activation lo * 2^11 into E4M3 against weight hi * 2^-12
        ah = E._f16(a)
        A[1] = E._e4((a - ah) * 2048.0) / 4096.0
    elif fault == "w_lo_last_block":                 # the weight lo plane read as zero in the last NB block
        nb = packing.conv_tc_block(c["w"].shape[2], 64 if fmt == "f8" else 128)
        W[2] = W[2].clone()
        W[2][..., -nb:] = 0.0
    elif fault == "seg0_header":                     # every K-segment scaled back with segment 0's 1/s
        taps, cin, _ = c["w"].shape
        s0 = E.weight_scale(c["w"][0:1, 0:seg_cin])
        f = torch.tensor([[E.weight_scale(c["w"][t:t + 1, k:k + seg_cin]) / s0 for k in range(0, cin, seg_cin)] for t in range(taps)])
        f = f.double().repeat_interleave(seg_cin, dim=1)[..., None]
        W = [w_ * f for w_ in W]
    acc = sum(E.conv1d(a_, w_, None, c["dil"], c["pad"]) for a_, w_ in zip(A, W))
    d = lambda t: None if t is None else t.double()
    return E.conv1d_epilogue(acc, d(c["bias"]), c["out_act"], 0.1, d(c["res"]), c["alpha"], d(c["y0"]), c["lens"])


FAULTS = [
    # fault, format, cases (variant, N) of the magnitude table
    ("lo_flush", "split3", [("x2^-12", 64), ("x2^-6", 64), ("x_chan2^-14..2^4", 64), ("x2^-12_epilogue", 64)]),
    ("f8_lo_2^11", "f8", [("x1", 64), ("x_chan2^-14..2^4", 64), ("cancel", 64)]),
    ("w_lo_last_block", "split3", [("x1", 192), ("w_outliers", 192)]),
    ("w_lo_last_block", "f8", [("x1", 192), ("w_outliers", 192)]),
]


@pytest.mark.parametrize("fault,fmt,cases", FAULTS, ids=[f"{f[0]}-{f[1]}" for f in FAULTS])
def test_fault_exceeds_bar(fault, fmt, cases):
    worst = 0.0
    for variant, N in cases:
        c = TC.mag_case(variant, N)
        y_c, y64, S, R = TC.contract(c, fmt)
        worst = max(worst, E.tc_errors(_fault_contract(c, fmt, fault), y_c, y64, S, R)[0])
        assert E.tc_errors(y_c, y_c, y64, S, R) == (0.0, 0.0)
    assert worst >= FAULT_FACTOR * E.TC_ACC_C, worst


def test_fault_segment_zero_header_exceeds_bar():
    worst = 0.0
    for case in TC.SEG_MAG_CASES:
        c = TC.seg_case(case)
        y_c, y64, S, R = TC.contract(c, "split3", seg_cin=packing.SEG_CIN)
        worst = max(worst, E.tc_errors(_fault_contract(c, "split3", "seg0_header", packing.SEG_CIN), y_c, y64, S, R)[0])
    assert worst >= FAULT_FACTOR * E.TC_SEG_ACC_C, worst


# A kernel that drops terms of its split: only the fp16 main term (the correction MMAs lost) or everything but the activation lo plane.
# Both must exceed the level-(a) bar by FAULT_FACTOR on EVERY shape of the tensor-core tests that carry that bar, long sums included
# (decoder conv-FFN, PostNet, HiFi-GAN ResBlock convs: up to 176 K-steps), in both formats.  Smallest factors at E.TC_ACC_C = 16:
# 10.1 on the LJSpeech checkpoint's stage-0 convs1.0 (f8), 13.5 over the test_gpu_ops shapes.
DROPS = ("hi_only", "a_lo_lost")


def _drop_scores(c, fmt, utts=None, seg_cin=None):
    """tc_errors (a) of the two dropped-term kernels of layer c."""
    sel = (lambda t: t) if utts is None else (lambda t: None if t is None else t[utts])
    y_c, y64, S, R = TC.contract(c, fmt, utts, seg_cin)
    terms = list(zip(E.a_planes(E.act_operand(sel(c["x"]), c["in_act"], 0.1), fmt), E._segmented(lambda v: E.w_planes(v, fmt), c["w"], seg_cin)))
    d = lambda t: None if t is None else t.double()
    out = []
    for kept in (terms[:1], [terms[0], terms[2]]):
        acc = sum(E.conv1d(a_, w_, None, c["dil"], c["pad"]) for a_, w_ in kept)
        yf = E.conv1d_epilogue(acc, d(c["bias"]), c["out_act"], 0.1, d(sel(c["res"])), c["alpha"], d(sel(c["y0"])), sel(c["lens"]))
        out.append(E.tc_errors(yf, y_c, y64, S, R)[0])
    return out


def _ops_layer(case):
    from tests import test_gpu_ops as G
    x, w, bias, res, y0, lens = G._conv_case(case)
    return dict(x=x, w=w, bias=bias, res=res, y0=y0, lens=lens, dil=case[5], pad=case[6], in_act=case[7], out_act=case[8], alpha=case[10])


def _tc_cases():
    from tests import test_gpu_ops as G
    return G.TC_CASES


@pytest.mark.parametrize("fmt", ["split3", "f8"])
@pytest.mark.parametrize("case", _tc_cases())
def test_dropped_terms_exceed_bar_tc_cases(case, fmt):
    """Every shape of test_conv1d_tensor_core / _f8_split, on the utterances those tests compare."""
    from tests import test_gpu_ops as G
    scores = _drop_scores(_ops_layer(case), fmt, G._ref_utts(case[0]))
    assert min(scores) >= FAULT_FACTOR * E.TC_ACC_C, dict(zip(DROPS, scores))


def test_dropped_terms_exceed_bar_segmented():
    """Every shape of test_conv1d_tensor_core_k_segmented and of the segmented magnitude table, against E.TC_SEG_ACC_C."""
    from tests import test_gpu_ops as G
    layers = []
    for case in G.SEG_CASES:
        x, w, bias, res, lens = G._seg_case(case)
        layers.append((dict(x=x, w=w, bias=bias, res=res, y0=None, lens=lens, dil=1, pad=case[5], in_act=case[6], out_act=0, alpha=1.0),
                       G._ref_utts(case[0])))
    layers += [(TC.seg_case(case), None) for case in TC.SEG_MAG_CASES]
    for c, utts in layers:
        if c["in_act"] == E.ACT_LRELU:                       # the encoder's ReLU input: leaky_relu with slope 0
            c = dict(c, x=torch.relu(c["x"]), in_act=E.ACT_NONE)
        scores = _drop_scores(c, "split3", utts, packing.SEG_CIN)
        assert min(scores) >= FAULT_FACTOR * E.TC_SEG_ACC_C, dict(zip(DROPS, scores))


@pytest.mark.parametrize("name", ["LJSpeech", "universal"])
def test_dropped_terms_exceed_bar_real_checkpoint(name):
    """Every layer test_real_checkpoint_layers runs through fs2_conv1d, in its format; and every fused ResBlock group it runs through
    fs2_resstack, whose single-pass fp16 version must exceed the fused-vs-unfused bar in every 128-row block."""
    import functools
    from oracle import real_ckpt
    from tests.test_gpu_tc_precision import RESSTACK_UNFUSED_C
    sd = real_ckpt.load(name)
    if sd is None:
        pytest.skip("real checkpoint fixture not present (run __graft_entry__.build() where the reference tree exists)")
    mel = torch.from_numpy(np.load(os.path.join(GOLD, f"hifigan_real_{name}.npz"))["mel"])[:1]
    convs, groups = TC.real_layers(*TC.hifigan_layer_inputs(sd, mel), TC.default_vocoder_masks())
    low = {key: min(_drop_scores(c, fmt)) for key, c, fmt in convs}
    assert min(low.values()) >= FAULT_FACTOR * E.TC_ACC_C, {k: v for k, v in low.items() if v < FAULT_FACTOR * E.TC_ACC_C}
    ks, ds = (3, 7, 11), ((1, 3, 5),) * 3
    for stage, x, w1, b1, w2, b2 in groups:
        full = E.resblock_group(x, ks, ds, w1, b1, w2, b2, conv=E.conv1d_f8)
        fp16 = E.resblock_group(x, ks, ds, w1, b1, w2, b2, conv=functools.partial(E.conv1d_f8, fp16_only=True))
        _, S, _ = E.resstack_contract(x, ks, ds, w1, b1, w2, b2)
        diff = (full - fp16).abs() / (E.U24 * S)
        blocks = [diff[0, s:s + 128].max().item() for s in range(0, x.shape[1], 128)]
        assert min(blocks) > FAULT_FACTOR * RESSTACK_UNFUSED_C, (stage, min(blocks))


# ------------------------------------------------------------------ activation headroom of the shipped checkpoints
# The f16 + f8 format saturates its correction from |a| = 256 on (lo * 2^12 leaves E4M3's range).  The generator's default policy
# (Generator.f8_mask) runs every upsample stage in that format: the phase-group convs and every ResBlock conv.  Largest |a| measured on
# the golden mels: LJSpeech 10.7, universal 23.2.
F8_HEADROOM = 256.0


@pytest.mark.parametrize("name", ["LJSpeech", "universal"])
def test_real_checkpoint_f8_activations_below_saturation(name):
    from oracle import real_ckpt
    sd = real_ckpt.load(name)
    if sd is None:
        pytest.skip("real checkpoint fixture not present (run __graft_entry__.build() where the reference tree exists)")
    mel = torch.from_numpy(np.load(os.path.join(GOLD, f"hifigan_real_{name}.npz"))["mel"])
    ins, _ = TC.hifigan_layer_inputs(sd, mel)
    lrelu = lambda t: torch.where(t > 0, t, 0.1 * t)
    peak = {k: lrelu(v).abs().max().item() for k, v in ins.items() if k != "conv_pre"}      # conv_pre runs the three-MMA split
    worst = max(peak, key=peak.get)
    assert peak[worst] < F8_HEADROOM, (worst, peak[worst])
