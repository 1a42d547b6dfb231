"""GPU: every C-ABI operator against its CPU contract (tests/emul_cabi.py, torch fp32 on CPU).  fp32 kernels: the only
difference allowed is summation order, so tolerances are a few ulp of the accumulated magnitude."""
import pytest
import torch

from fastspeech2_b200 import ops, packing
from tests import emul_cabi as E

pytestmark = pytest.mark.gpu
DEV = "cuda"


def g(seed=0):
    return torch.Generator().manual_seed(seed)


def rnd(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=g(seed)) * scale


CONV_CASES = [
    # B, T, Cin, N, taps, dil, pad, in_act, out_act, res, alpha, accumulate, lens
    (2, 200, 256, 768, 1, 1, 0, 0, 0, False, 1.0, False, False),     # QKV projection
    (2, 131, 256, 1024, 9, 1, 4, 0, 1, False, 1.0, False, False),    # conv-FFN w_1 + ReLU
    (2, 131, 1024, 256, 1, 1, 0, 0, 0, True, 1.0, False, False),     # conv-FFN w_2 + residual
    (3, 77, 80, 512, 5, 1, 2, 0, 2, False, 1.0, False, False),       # PostNet first conv + tanh
    (3, 77, 512, 80, 5, 1, 2, 0, 0, True, 1.0, False, False),        # PostNet last conv + mel residual (N = 80)
    (1, 300, 128, 128, 11, 5, 25, 3, 3, False, 1.0, False, False),   # HiFi-GAN resblock conv1 (dilated, lrelu in/out)
    (2, 260, 64, 64, 7, 1, 3, 0, 0, True, 1.0 / 3, True, False),     # resblock conv2 accumulate into stage sum
    (2, 515, 32, 32, 3, 3, 3, 3, 3, False, 1.0, False, False),       # last stage, N = 32
    (2, 140, 256, 256, 3, 1, 1, 0, 1, False, 1.0, False, True),      # with row masking
    (1, 1, 256, 256, 3, 1, 1, 0, 0, False, 1.0, False, False),       # single row
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv1d(case):
    B, T, Cin, N, taps, dil, pad, in_act, out_act, use_res, alpha, acc, use_lens = case
    x = rnd(B, T, Cin, seed=1)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    res = rnd(B, T, N, seed=4) if use_res else None
    y0 = rnd(B, T, N, seed=5) if acc else None
    lens = torch.tensor([max(1, T - 7 * (i + 1)) for i in range(B)], dtype=torch.int32) if use_lens else None
    want = E.conv1d(x, w, bias, dil, pad, in_act, 0.1, out_act, 0.1, res, alpha, y0, lens)
    out = y0.to(DEV).clone() if acc else None
    got = ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), dilation=dil, pad_left=pad, in_act=in_act, in_slope=0.1, out_act=out_act,
                     out_slope=0.1, res=None if res is None else res.to(DEV), alpha=alpha, out=out, accumulate=acc,
                     row_lens=None if lens is None else lens.to(DEV))
    torch.cuda.synchronize()
    err = (got.cpu() - want).abs().max().item()
    assert err < 2e-5, err


TC_CASES = [
    # B, T, Cin, N, taps, dil, pad, in_act, out_act, res, alpha, accumulate, lens      (tensor-core split-FP16 kernel, backend = 2)
    (1, 128, 16, 128, 1, 1, 0, 0, 0, False, 1.0, False, False),      # one tile, one K-block
    (2, 300, 64, 128, 3, 1, 1, 0, 0, False, 1.0, False, False),      # ragged tail tile
    (2, 700, 128, 128, 11, 5, 25, 3, 3, True, 1.0, False, False),    # HiFi-GAN stage-1 conv1 shape: dilation 5, lrelu in/out
    (2, 520, 256, 256, 7, 1, 3, 0, 0, True, 1.0 / 3, True, False),   # two N-blocks, residual + scaled accumulate
    (2, 333, 512, 80, 5, 1, 2, 0, 0, True, 1.0, False, False),       # PostNet last conv: N = 80 (16-column tail block)
    (2, 260, 256, 1024, 9, 1, 4, 0, 1, False, 1.0, False, False),    # conv-FFN w_1 + ReLU, 8 N-blocks
    (3, 200, 1024, 256, 1, 1, 0, 0, 0, True, 1.0, False, True),      # conv-FFN w_2 + residual + pad-row mask
    (2, 1500, 32, 32, 3, 3, 3, 3, 3, False, 1.0, False, False),      # 32 channels: two accumulator groups
    (2, 777, 64, 64, 7, 1, 3, 3, 0, True, 1.0, False, False),        # 64 channels: two accumulator groups
    (2, 150, 80, 512, 7, 1, 3, 0, 0, False, 1.0, False, False),      # conv_pre: C_in = 80
    (2, 257, 64, 64, 2, 1, 1, 3, 0, False, 1.0, False, False),       # ConvTranspose phase group (2 taps)
    (1, 40, 256, 80, 1, 1, 0, 0, 2, False, 1.0, False, False),       # short sequence, tanh epilogue
]


@pytest.mark.parametrize("case", TC_CASES)
def test_conv1d_tensor_core(case):
    """fs2_conv1d through the tensor-core kernel against an fp64 evaluation of the same contract.  Error budget: the split
    keeps 22 bits; what remains is the tensor core's truncating fp32 accumulator (~0.5 ulp per K=16 step)."""
    B, T, Cin, N, taps, dil, pad, in_act, out_act, use_res, alpha, acc, use_lens = case
    x = rnd(B, T, Cin, seed=1)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    res = rnd(B, T, N, seed=4) if use_res else None
    y0 = rnd(B, T, N, seed=5) if acc else None
    lens = torch.tensor([max(1, T - 7 * (i + 1)) for i in range(B)], dtype=torch.int32) if use_lens else None
    d = lambda t: None if t is None else t.double()
    want = E.conv1d(x.double(), w.double(), bias.double(), dil, pad, in_act, 0.1, out_act, 0.1, d(res), alpha, d(y0), lens)
    wtc = packing.pack_conv_tc(w)
    assert wtc is not None
    out = y0.to(DEV).clone() if acc else None
    got = ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), dilation=dil, pad_left=pad, in_act=in_act, in_slope=0.1, out_act=out_act,
                     out_slope=0.1, res=None if res is None else res.to(DEV), alpha=alpha, out=out, accumulate=acc,
                     row_lens=None if lens is None else lens.to(DEV), w_tc=wtc.to(DEV), backend=2)
    torch.cuda.synchronize()
    err = (got.cpu().double() - want).abs().max().item()
    assert err < 6e-5, err


def _f8_operand_emulation(x, w, in_act, in_slope):
    """The operands the f16 + f8 kernel multiplies, evaluated exactly: returns (a_hi, w_hi, a_lo8, w_hi8, a_hi8, w_lo8, scale) in fp64
    so that  y*scale = a_hi.w_hi + a_lo8.w_hi8 + a_hi8.w_lo8  (conv_tc_kernel.cuh::tc_convert_store, packing.pack_conv_tc)."""
    e4 = lambda t: t.float().clamp(-448, 448).to(torch.float8_e4m3fn).double()
    a = x.float()
    if in_act == 3:
        a = torch.maximum(a, a * in_slope)
    ah = a.half().float()
    al = a - ah
    hi, _, s = packing.split_fp16(w)
    wl = w.float() * s - hi.float()
    return (ah.double(), hi.double(), e4(al * 4096.0) / 4096.0, e4(hi.float() * 2.0 ** -12) * 4096.0, e4(ah), e4(wl), s)


@pytest.mark.parametrize("case", TC_CASES)
def test_conv1d_tensor_core_f8_split(case):
    """FS2_TC_VARIANT_F8 (fp16 main term + one E4M3 correction MMA): (a) the kernel computes exactly the rounded-operand products of
    its contract (checked against an fp64 evaluation of those operands, so a wrong byte order / scale / K layout cannot hide),
    (b) against the unrounded fp64 contract the error is at the 2^-16 level (budget for the parity bars: scripts/emul_split_precision.py)."""
    B, T, Cin, N, taps, dil, pad, in_act, out_act, use_res, alpha, acc, use_lens = case
    x = rnd(B, T, Cin, seed=1)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    res = rnd(B, T, N, seed=4) if use_res else None
    y0 = rnd(B, T, N, seed=5) if acc else None
    lens = torch.tensor([max(1, T - 7 * (i + 1)) for i in range(B)], dtype=torch.int32) if use_lens else None
    d = lambda t: None if t is None else t.double()
    exact = E.conv1d(x.double(), w.double(), bias.double(), dil, pad, in_act, 0.1, out_act, 0.1, d(res), alpha, d(y0), lens)
    ah, wh, al8, wh8, ah8, wl8, s = _f8_operand_emulation(x, w, in_act, 0.1)
    lin = lambda a_, w_: E.conv1d(a_, w_, None, dil, pad, 0, 0.0, 0, 0.0, None, 1.0, None, None)
    pre = (lin(ah, wh) + lin(al8, wh8) + lin(ah8, wl8)) / s                       # pre-activation, no bias
    want = E.conv1d_epilogue(pre, bias.double(), out_act, 0.1, d(res), alpha, d(y0), lens)
    wtc = packing.pack_conv_tc(w, f8=True)
    out = y0.to(DEV).clone() if acc else None
    got = ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), dilation=dil, pad_left=pad, in_act=in_act, in_slope=0.1, out_act=out_act,
                     out_slope=0.1, res=None if res is None else res.to(DEV), alpha=alpha, out=out, accumulate=acc,
                     row_lens=None if lens is None else lens.to(DEV), w_tc=wtc.to(DEV), backend=2, tc_variant=1)
    torch.cuda.synchronize()
    err_contract = (got.cpu().double() - want).abs().max().item()
    err_exact = (got.cpu().double() - exact).abs().max().item()
    assert err_contract < 6e-5, (err_contract, err_exact)      # same budget as the three-MMA split: only the accumulator's rounding
    assert err_exact < 1.5e-3, (err_contract, err_exact)       # ~2^-16 relative on O(1..10) outputs (single-pass fp16: ~2e-2 here)


SEG_CASES = [
    # B, T, Cin, N, taps, pad, in_act (0 none / 3 = lrelu slope 0 = ReLU), res, lens
    (2, 128, 256, 768, 1, 0, 0, False, False),      # encoder QKV projection
    (3, 100, 256, 1024, 9, 4, 0, False, False),     # conv-FFN w_1 (pre-activation output)
    (2, 128, 1024, 256, 1, 0, 3, True, True),       # conv-FFN w_2: ReLU on the input, residual, pad-row mask, 4 channel chunks
    (2, 300, 256, 256, 3, 1, 0, False, False),      # predictor conv, T > 256 (several tiles per utterance)
]


@pytest.mark.parametrize("case", SEG_CASES)
def test_conv1d_tensor_core_k_segmented(case):
    """FS2_TC_VARIANT_NB64 | FS2_TC_VARIANT_SEGMENTED: one launch whose work units are (tile, tap, 256-channel chunk) slices with fresh
    16-step accumulators, summed in fp32 through y.  Against the fp64 contract the error must be at the fp32 kernel's level (the point
    of the segmentation: a single 432-step accumulation leaves 5x more)."""
    B, T, Cin, N, taps, pad, in_act, use_res, use_lens = case
    x = rnd(B, T, Cin, seed=1)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    res = rnd(B, T, N, seed=4) if use_res else None
    lens = torch.tensor([max(1, T - 7 * (i + 1)) for i in range(B)], dtype=torch.int32) if use_lens else None
    d = lambda t: None if t is None else t.double()
    want = E.conv1d(x.double(), w.double(), bias.double(), 1, pad, in_act, 0.0, 0, 0.0, d(res), 1.0, None, lens)
    wseg = packing.pack_conv_tc_segments(w)
    assert wseg is not None and wseg.numel() == taps * (Cin // 256) * (128 + 1024 * N)
    got = ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), pad_left=pad, in_act=in_act, in_slope=0.0, res=None if res is None else res.to(DEV),
                     row_lens=None if lens is None else lens.to(DEV), w_tc=wseg.to(DEV), backend=2, tc_variant=2 | 4)
    exact = ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), pad_left=pad, in_act=in_act, in_slope=0.0, res=None if res is None else res.to(DEV),
                       row_lens=None if lens is None else lens.to(DEV), backend=1)
    torch.cuda.synchronize()
    err = (got.cpu().double() - want).abs().max().item()
    err_fp32 = (exact.cpu().double() - want).abs().max().item()
    assert err < 4e-6 and err < 4 * err_fp32 + 1e-6, (err, err_fp32)


RESSTACK_CASES = [
    # B, N, C, kernels, dilations
    (1, 700, 32, (3, 7, 11), ((1, 3, 5),) * 3),       # two work items, ragged second tile
    (2, 392 * 2, 32, (3, 7, 11), ((1, 3, 5),) * 3),   # exact multiple of the tile
    (2, 100, 32, (3, 7, 11), ((1, 3, 5),) * 3),       # utterance shorter than the halo-extended slab
    (2, 900, 64, (3, 7, 11), ((1, 3, 5),) * 3),       # 64 channels: three 128-row tiles per slab
    (1, 264, 64, (3, 7, 11), ((1, 3, 5),) * 3),       # exactly one tile
    (3, 50, 64, (3, 5), ((1, 2), (2, 6))),            # other kernel sets / dilation lists
]


@pytest.mark.parametrize("case", RESSTACK_CASES)
def test_resstack_fused(case):
    """fs2_resstack (one persistent kernel for a whole multi-receptive-field ResBlock group, intermediates on chip, halo recompute)
    against an fp64 evaluation of hifigan/models.py:96-103,:154-160 with torch conv1d.  Error budget: the f16 + f8 operand split
    (2^-16 relative per layer) through 6 layers per kernel size."""
    import torch.nn.functional as F
    B, N, C, kernels, dils = case
    x = rnd(B, N, C, seed=21)
    w1, b1, w2, b2 = [], [], [], []
    want = torch.zeros(B, C, N, dtype=torch.float64)
    for j, k in enumerate(kernels):
        w1.append([]); b1.append([]); w2.append([]); b2.append([])
        r = x.double().transpose(1, 2)
        for d, dv in enumerate(dils[j]):
            wa = rnd(C, C, k, seed=100 + 10 * j + d, scale=0.6 * (C * k) ** -0.5)      # [out, in, k]
            wb = rnd(C, C, k, seed=200 + 10 * j + d, scale=0.6 * (C * k) ** -0.5)
            ba, bb = rnd(C, seed=300 + 10 * j + d, scale=0.05), rnd(C, seed=400 + 10 * j + d, scale=0.05)
            t = F.conv1d(F.leaky_relu(r, 0.1), wa.double(), ba.double(), dilation=dv, padding=(k - 1) * dv // 2)
            t = F.conv1d(F.leaky_relu(t, 0.1), wb.double(), bb.double(), padding=(k - 1) // 2)
            r = t + r
            w1[j].append(packing.pack_conv_tc(packing.conv_w(wa), f8=True).to(DEV)); b1[j].append(ba.to(DEV))
            w2[j].append(packing.pack_conv_tc(packing.conv_w(wb), f8=True).to(DEV)); b2[j].append(bb.to(DEV))
        want += r
    want = (want / len(kernels)).transpose(1, 2)
    got = ops.resstack(x.to(DEV), kernels, dils, w1, b1, w2, b2)
    torch.cuda.synchronize()
    err = (got.cpu().double() - want).abs().max().item()
    assert torch.isfinite(got).all()
    assert err < 3e-4 * max(1.0, want.abs().max().item()), (err, want.abs().max().item())


@pytest.mark.parametrize("C,k,dils,N", [(64, 3, (5,), 1000), (64, 7, (3,), 1000), (32, 3, (1,), 1000), (64, 11, (5,), 777), (32, 11, (5,), 1500),
                                        (32, 7, (3,), 900), (64, 3, (1, 3, 5), 1234), (64, 3, (1,), 21000), (32, 7, (1,), 40000), (64, 5, (2,), 40)])
def test_resstack_single_pair_accumulate(C, k, dils, N):
    """The single-kernel-size mode of fs2_resstack (n_kernels = 1, alpha, accumulate): y += alpha * ResBlock_k,dils(x).  With a small
    halo the kernel runs independent 128-row tiles (each with its own halo) and prefetches the next work item's input; the long cases
    give every CTA several work items."""
    import torch.nn.functional as F
    B = 2
    x = rnd(B, N, C, seed=41)
    y0 = rnd(B, N, C, seed=42)
    r = x.double().transpose(1, 2)
    w1, b1, w2, b2 = [], [], [], []
    for i, dil in enumerate(dils):
        wa = rnd(C, C, k, seed=43 + 10 * i, scale=0.6 * (C * k) ** -0.5); wb = rnd(C, C, k, seed=44 + 10 * i, scale=0.6 * (C * k) ** -0.5)
        ba, bb = rnd(C, seed=45 + 10 * i, scale=0.05), rnd(C, seed=46 + 10 * i, scale=0.05)
        t = F.conv1d(F.leaky_relu(r, 0.1), wa.double(), ba.double(), dilation=dil, padding=(k - 1) * dil // 2)
        t = F.conv1d(F.leaky_relu(t, 0.1), wb.double(), bb.double(), padding=(k - 1) // 2)
        r = t + r
        w1.append(packing.pack_conv_tc(packing.conv_w(wa), f8=True).to(DEV)); b1.append(ba.to(DEV))
        w2.append(packing.pack_conv_tc(packing.conv_w(wb), f8=True).to(DEV)); b2.append(bb.to(DEV))
    want = y0.double() + (1.0 / 3) * r.transpose(1, 2)
    out = y0.to(DEV).clone()
    ops.resstack(x.to(DEV), (k,), (tuple(dils),), [w1], [b1], [w2], [b2], alpha=1.0 / 3, out=out, accumulate=True)
    torch.cuda.synchronize()
    err = (out.cpu().double() - want).abs().max().item()
    assert torch.isfinite(out).all()
    assert err < 1e-4 * len(dils) * max(1.0, want.abs().max().item()), err


def test_conv1d_tensor_core_alignment_contract():
    """The tensor-core kernel reads activations with 256-bit loads: a 16-byte-but-not-32-byte aligned x is refused by the explicit
    backend and silently served by the exact fp32 kernel under FS2_CONV_AUTO (same contract, fp32 accuracy)."""
    from fastspeech2_b200._lib import Fs2Error
    B, T, Cin, N = 2, 200, 64, 64
    buf = rnd(B * T * Cin + 8, seed=11).to(DEV)
    x = buf[4:4 + B * T * Cin].view(B, T, Cin)
    assert x.data_ptr() % 32 == 16
    w = rnd(3, Cin, N, seed=12, scale=0.1)
    wtc = packing.pack_conv_tc(w).to(DEV)
    with pytest.raises(Fs2Error):
        ops.conv1d(x, w.to(DEV), None, pad_left=1, w_tc=wtc, backend=2)
    got = ops.conv1d(x, w.to(DEV), None, pad_left=1, w_tc=wtc, backend=0)
    torch.cuda.synchronize()
    want = E.conv1d(x.cpu().double(), w.double(), None, 1, 1, 0, 0.0, 0, 0.0, None, 1.0, None, None)
    assert (got.cpu().double() - want).abs().max().item() < 5e-6


def test_conv1d_tensor_core_large_activations():
    """|x| beyond the fp16 range saturates in the hi/lo split instead of turning into inf / NaN (hi = 65504, lo = fp16(x - hi))."""
    B, T, Cin, N = 1, 128, 16, 16
    x = rnd(B, T, Cin, seed=13)
    x[0, 5, 3] = 7.0e4; x[0, 9, 0] = -9.0e4
    w = rnd(1, Cin, N, seed=14, scale=0.1)
    got = ops.conv1d(x.to(DEV), w.to(DEV), None, w_tc=packing.pack_conv_tc(w).to(DEV), backend=2)
    torch.cuda.synchronize()
    want = E.conv1d(x.double(), w.double(), None, 1, 0, 0, 0.0, 0, 0.0, None, 1.0, None, None)
    assert torch.isfinite(got).all()
    assert (got.cpu().double() - want).abs().max().item() < 2e-3 * want.abs().max().item()


def test_conv1d_strided_output_conv_transpose():
    for u, cin, cout, T in ((8, 64, 32, 37), (2, 64, 32, 130)):
        w = rnd(cin, cout, 2 * u, seed=7, scale=0.1)
        x = rnd(2, T, cin, seed=8)
        bias = rnd(cout, seed=9, scale=0.1)
        want = torch.nn.functional.conv_transpose1d(torch.nn.functional.leaky_relu(x, 0.1).transpose(1, 2), w, bias, stride=u,
                                                    padding=u // 2).transpose(1, 2)
        wa, wb = packing.split_conv_transpose(w, u)
        half = u // 2
        out = torch.empty(2, T, u * cout, device=DEV)
        bt = bias.repeat(u).to(DEV)
        xd = x.to(DEV)
        ops.conv1d(xd, wa.to(DEV), bt[: half * cout], pad_left=1, in_act=3, in_slope=0.1, out=out[:, :, : half * cout])
        ops.conv1d(xd, wb.to(DEV), bt[half * cout:], pad_left=0, in_act=3, in_slope=0.1, out=out[:, :, half * cout:])
        torch.cuda.synchronize()
        err = (out.cpu().reshape(2, T * u, cout) - want).abs().max().item()
        assert err < 2e-5, err


def test_conv1d_rejects_bad_shapes():
    from fastspeech2_b200._lib import Fs2Error
    x = torch.zeros(1, 8, 24, device=DEV)          # Cin % 16 != 0
    w = torch.zeros(1, 24, 16, device=DEV)
    with pytest.raises(Fs2Error):
        ops.conv1d(x, w)


@pytest.mark.parametrize("C", [256, 512, 1024, 80])
def test_layernorm(C):
    x = rnd(3, 50, C, seed=1, scale=3.0) + 0.5
    gm, bt = 1 + rnd(C, seed=2, scale=0.1), rnd(C, seed=3, scale=0.1)
    lens = torch.tensor([50, 13, 1], dtype=torch.int32)
    for ln_ in (None, lens):
        want = E.layernorm(x, gm, bt, ln_)
        got = ops.layernorm(x.to(DEV), gm.to(DEV), bt.to(DEV), None if ln_ is None else ln_.to(DEV))
        assert (got.cpu() - want).abs().max() < 5e-6


@pytest.mark.parametrize("T,lens", [(130, [130, 64, 1]), (64, [64, 64, 33]), (257, [257, 200, 65])])
def test_attention(T, lens):
    qkv = rnd(3, T, 768, seed=1)
    kl = torch.tensor(lens, dtype=torch.int32)
    want = E.attention(qkv, 2, kl)
    got = ops.attention(qkv.to(DEV), 2, kl.to(DEV))
    torch.cuda.synchronize()
    assert (got.cpu() - want).abs().max() < 5e-6


@pytest.mark.parametrize("T,lens", [(300, [300, 129, 1]), (1000, [1000, 777, 513]), (1100, [1100, 64, 1037])])
def test_attention_tensor_core_path(T, lens):
    """S = QK^T / PV as split-FP16 tensor-core GEMMs + row softmax (decoder path): fp32-class accuracy expected."""
    qkv = rnd(3, T, 768, seed=2)
    kl = torch.tensor(lens, dtype=torch.int32)
    want = E.attention(qkv.double(), 2, kl)
    got = ops.attention(qkv.to(DEV), 2, kl.to(DEV), backend=1)
    exact = ops.attention(qkv.to(DEV), 2, kl.to(DEV), backend=0)
    torch.cuda.synchronize()
    err = (got.cpu().double() - want).abs().max().item()
    err0 = (exact.cpu().double() - want).abs().max().item()
    assert err < 2e-5, (err, err0)


@pytest.mark.parametrize("T,lens", [(128, [128, 5, 77]), (300, [300, 129, 1]), (1017, [1017, 777, 513]), (1100, [1100, 64, 1037]), (4200, [4200, 4097, 9])])
def test_attention_fused_kernel(T, lens):
    """fs2_attention backend 2: QK^T, softmax and PV in ONE tensor-core kernel (scores stay in registers; two-pass softmax; no length
    limit) against an fp64 evaluation of transformer/Modules.py:14-25 with the key mask of Models.py:79.  Same budget as the GEMM path."""
    qkv = rnd(3, T, 768, seed=3)
    kl = torch.tensor(lens, dtype=torch.int32)
    want = E.attention(qkv.double(), 2, kl)
    got = ops.attention(qkv.to(DEV), 2, kl.to(DEV), backend=2)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    err = (got.cpu().double() - want).abs().max().item()
    assert err < 2e-5, err
    # padded query rows are written as exact zeros (contract of fs2_attention)
    for b, n in enumerate(lens):
        assert (got[b, n:] == 0).all()


def test_embed_and_speaker():
    table = rnd(361, 256, seed=1)
    pos = rnd(1001, 256, seed=2)
    ids = torch.randint(0, 361, (4, 37), generator=g(3))
    y = ops.embed_positions(ids.to(DEV), table.to(DEV), pos.to(DEV))
    assert torch.equal(y.cpu(), table[ids] + pos[:37])
    spk = rnd(904, 256, seed=4)
    sid = torch.randint(0, 904, (4,), generator=g(5))
    y2 = ops.add_speaker_(y.clone(), spk.to(DEV), sid.to(DEV))
    assert torch.equal(y2.cpu(), (table[ids] + pos[:37]) + spk[sid][:, None, :])


def test_variance_head():
    h = rnd(3, 40, 256, seed=1)
    w, b = rnd(256, seed=2, scale=0.1), torch.tensor([0.3])
    lens = torch.tensor([40, 25, 3], dtype=torch.int32)
    bins = torch.linspace(-2.9, 11.4, 255)
    emb = rnd(256, 256, seed=3)
    x = rnd(3, 40, 256, seed=4)
    tgt = rnd(3, 40, seed=5, scale=3.0)
    # duration-style (no bins)
    want, _ = E.variance_head(h, w, b, lens, 1.0, None, None, None, None)
    got = ops.variance_head(h.to(DEV), w.to(DEV), b.to(DEV), lens.to(DEV))
    assert (got.cpu() - want).abs().max() < 2e-6
    for target, control in ((None, 1.3), (tgt, 1.0)):
        wp, wx = E.variance_head(h, w, b, lens, control, target, bins, emb, x)
        xd = x.to(DEV).clone()
        gp = ops.variance_head(h.to(DEV), w.to(DEV), b.to(DEV), lens.to(DEV), control, None if target is None else target.to(DEV),
                               bins.to(DEV), emb.to(DEV), xd)
        assert (gp.cpu() - wp).abs().max() < 2e-6
        assert (xd.cpu() - wx).abs().max() < 1e-6     # same buckets picked


def test_bucketize_edges_exact():
    """torch.bucketize(right=False): a value equal to an edge goes to that edge's index."""
    bins = torch.linspace(-1.0, 1.0, 255)
    vals = torch.cat([bins[[0, 1, 100, 254]], torch.tensor([-5.0, 5.0, 0.0])])
    n = vals.numel()
    h = torch.zeros(1, n, 4); h[0, :, 0] = vals
    w = torch.tensor([1.0, 0, 0, 0]); b = torch.zeros(1)
    emb = torch.arange(256, dtype=torch.float32)[:, None].repeat(1, 4)
    x = torch.zeros(1, n, 4, device=DEV)
    ops.variance_head(h.to(DEV), w.to(DEV), b.to(DEV), None, 1.0, None, bins.to(DEV), emb.to(DEV), x)
    assert torch.equal(x[0, :, 0].cpu().long(), torch.bucketize(vals, bins))


@pytest.mark.parametrize("L,d_control", [(40, 1.0), (300, 2.5), (1000, 0.7)])
def test_durations_and_length_regulate(L, d_control):
    B = 3
    logd = rnd(B, L, seed=1, scale=0.6) + 1.2
    logd[1, L // 2:] = 0.0                                    # padded phonemes predict log-duration 0 -> d = 0
    logd[0, :5] = torch.log(torch.tensor([3.5, 4.5, 1.5, 2.5, 1.0]))   # round-half-even cases
    wd, wcum, wlen = E.durations(logd, False, d_control)
    d, cum, mel_lens, mel_lens32, stats = ops.durations(logd.to(DEV), False, d_control)
    assert torch.equal(d.cpu(), wd) and torch.equal(cum.cpu(), wcum) and torch.equal(mel_lens.cpu(), wlen)
    assert stats.cpu().tolist() == [int(wlen.max()), int(wlen.sum()), 0]          # max, sum, count of non-finite durations
    x = rnd(B, L, 256, seed=2)
    pos = rnd(int(wlen.max()) + 8, 256, seed=3)
    for T in (int(wlen.max()), int(wlen.max()) + 5):
        want = E.length_regulate(x, wcum, pos, T)
        got = ops.length_regulate(x.to(DEV), cum, T, pos.to(DEV))
        assert torch.equal(got.cpu(), want)                   # gather + one add: bit exact
    # integer targets (teacher forcing)
    tgt = torch.randint(0, 9, (B, L), generator=g(4)).float()
    _, wcum2, wlen2 = E.durations(tgt, True, 1.0)
    _, cum2, ml2, _, _ = ops.durations(tgt.to(DEV), True, 1.0)
    assert torch.equal(cum2.cpu(), wcum2) and torch.equal(ml2.cpu(), wlen2)


def test_conv_post_and_transpose():
    """lrelu -> Conv1d(C, 1, k) -> tanh (hifigan/models.py:161-163).  C = 32, k = 7 runs the register-resident kernel (8 lanes per row,
    sliding accumulators, 120 output rows per lane group: lengths around the group and 8-sample store boundaries); anything else the
    shared-memory kernel."""
    for B, T, C, k in ((2, 700, 32, 7), (3, 1, 32, 7), (1, 5, 32, 7), (2, 119, 32, 7), (2, 120, 32, 7), (3, 121, 32, 7), (1, 12345, 32, 7),
                       (5, 963, 32, 7), (2, 300, 16, 5), (2, 130, 32, 3)):
        x = rnd(B, T, C, seed=1 + T)
        w = rnd(k, C, seed=2, scale=0.1)
        b = torch.tensor([0.05])
        xa = torch.where(x > 0, x, x * 0.01).double()
        want = torch.tanh(torch.nn.functional.conv1d(xa.transpose(1, 2), w.double().t()[None], b.double(), padding=(k - 1) // 2))[:, 0]
        got = ops.conv_post(x.to(DEV), w.to(DEV), b.to(DEV), 0.01)
        assert got.shape == (B, T) and (got.cpu().double() - want).abs().max() < 2e-6, (B, T, C, k)
    m = rnd(3, 80, 45, seed=3)
    assert torch.equal(ops.transpose_bct_to_btc(m.to(DEV)).cpu(), m.transpose(1, 2).contiguous())
