"""GPU: every C-ABI operator against its CPU contract (tests/emul_cabi.py, torch fp32 on CPU).  fp32 kernels: the only
difference allowed is summation order, so tolerances are a few ulp of the accumulated magnitude."""
import pytest
import torch

from fastspeech2_b200 import ops, packing
from tests import emul_cabi as E
from tests.att_cases import ATT_EXACT_C, EDGE_LENS, attention_bar_scale, attention_normalised_err, attention_qkv

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
    # every (BM, BN) tile of the exact kernel (fs2_conv_simt_plan on 132 SMs, noted per group; tests/test_abi.py checks it), each with
    # all four output activations, T % BM != 0 and N % BN != 0.  A trailing dict sets in_slope (default 0.1) or strided views.
    # (128, 128)
    (16, 1000, 256, 1024, 9, 1, 4, 0, 1, False, 1.0, False, True),   # decoder conv-FFN w_1 + ReLU at B = 16
    (2, 17000, 16, 80, 3, 2, 1, 3, 2, False, 1.0, False, False),     # N = 80, off-centre pad, lrelu in, tanh
    (6, 2100, 64, 336, 3, 1, 1, 3, 3, True, -0.5, True, False),      # N = 336, residual, negative alpha, accumulate
    (2, 8500, 32, 208, 1, 1, 0, 0, 0, True, 0.5, True, False, {"strided": True}),
    # (128, 64)
    (2, 17000, 16, 48, 5, 3, 6, 3, 0, True, 1.0, False, False, {"in_slope": 0.0}),
    (4, 8500, 64, 64, 7, 1, 3, 0, 1, False, 1.0, False, True),
    (3, 12000, 32, 48, 11, 5, 25, 3, 3, False, 1.0, False, False),   # 11 taps, dilation 5
    (2, 17000, 16, 64, 1, 1, 0, 0, 2, False, 1.0, True, False),
    # (128, 32): two-column stores (GW = 2)
    (2, 17000, 32, 20, 3, 1, 1, 3, 0, False, 1.0, False, False, {"strided": True}),
    (2, 17000, 16, 32, 7, 2, 0, 0, 1, False, 1.0, False, True),      # pad_left 0
    (2, 17000, 32, 32, 3, 3, 3, 3, 3, True, 1.0 / 3, True, False),
    (2, 17000, 16, 12, 1, 1, 0, 0, 2, False, 1.0, True, False),
    # (64, 128)
    (2, 1500, 64, 336, 3, 1, 1, 0, 0, True, 1.0, False, True),
    (4, 1100, 256, 256, 3, 1, 1, 0, 1, False, 1.0, False, True),
    (4, 1100, 80, 512, 5, 1, 2, 0, 2, False, 1.0, False, False),     # PostNet first conv + tanh
    (2, 2200, 128, 208, 11, 5, 25, 3, 3, True, 1.0, False, False, {"strided": True}),
    # (64, 64)
    (2, 300, 64, 48, 5, 2, 4, 3, 3, False, 1.0, False, False, {"in_slope": 0.0}),
    (3, 200, 16, 48, 3, 1, 1, 0, 1, False, 1.0, False, False),
    (2, 100, 512, 80, 5, 1, 2, 0, 2, True, 1.0, True, True),
    (2, 150, 1024, 64, 9, 1, 4, 0, 0, False, 1.0, False, False),     # K = 9216, the longest sum in the table
    # (64, 32)
    (2, 200, 16, 20, 3, 1, 1, 3, 0, True, 1.0, False, True, {"in_slope": 0.0}),
    (1, 1, 16, 32, 3, 1, 1, 0, 1, False, 1.0, False, False),         # T = 1, one K-step per tap
    (2, 77, 16, 4, 1, 1, 0, 0, 2, False, 2.0, True, False),          # N = 4
]
SIMT_TILES = {(bm, bn) for bm in (64, 128) for bn in (32, 64, 128)}

# |y - y64| <= CONV_EXACT_C * 2^-24 * scale per element, scale = |alpha| (sum |in_act(x)| |w| + |bias| + |res|) + |y0|: what fp32
# summation in any order can lose, so the bar scales with the sum instead of being loose at small K and tight at large K.  Largest
# value measured over CONV_CASES and RAGGED_CONV_CASES on an H100 80GB HBM3 (700 W power limit): 8.6, so the bar leaves 4.2x headroom.
CONV_EXACT_C = 36.0
U24 = 2.0 ** -24


def _case_opts(case):
    return (case[:-1], case[-1]) if isinstance(case[-1], dict) else (case, {})


def simt_plan(B, T, Cin, N, taps, num_sms=132):
    """fs2_conv_simt_plan: the (BM, BN) tile the exact kernel takes for this shape on num_sms SMs (host logic, no GPU needed)."""
    import ctypes
    from fastspeech2_b200 import _lib as L
    a = L.Conv1dArgs(x=16, w=16, y=16, B=B, T=T, Cin=Cin, N=N, taps=taps, alpha=1.0)
    out = L.ConvSimtPlan()
    assert L.lib().fs2_conv_simt_plan(ctypes.byref(a), num_sms, ctypes.byref(out)) == 0
    return out.BM, out.BN


def conv_scale(x, w, bias, dil, pad, in_act, in_slope, res, alpha, y0, lens):
    """The scale of the exact conv's bar: the same fp64 contract evaluated on absolute values."""
    a = lambda t: None if t is None else t.double().abs()
    return E.conv1d(E._act(x.double(), in_act, in_slope).abs(), a(w), a(bias), dil, pad, 0, 0.0, 0, 0.0, a(res), abs(alpha), a(y0), lens)


def normalised_err(got, want, scale):
    """max |got - want| / (2^-24 scale); where scale = 0 (masked rows) the output must be exact."""
    d = (got.double() - want).abs()
    r = torch.where(scale > 0, d / (U24 * scale.clamp_min(1e-300)), torch.where(d > 0, float("inf"), 0.0))
    return torch.nan_to_num(r, nan=float("inf")).max().item()


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv1d(case, parity_log):
    """fs2_conv1d through the exact fp32 kernel (backend 1), every utterance, against an fp64 evaluation of the same contract, within a
    bar that scales with the accumulated magnitude."""
    case, opts = _case_opts(case)
    B, T, Cin, N, taps, dil, pad, in_act, out_act, use_res, alpha, acc, _ = case
    slope = opts.get("in_slope", 0.1)
    x, w, bias, res, y0, lens = _conv_case(case)
    dv = lambda t: None if t is None else t.to(DEV)
    xd, rd, yd = dv(x), dv(res), dv(y0)
    if opts.get("strided"):           # x, res and y as channel slices of wider buffers
        xd = torch.full((B, T, Cin + 24), float("nan"), device=DEV)[:, :, 8:8 + Cin]
        xd.copy_(x)
        if res is not None:
            rd = torch.full((B, T, N + 40), float("nan"), device=DEV)[:, :, 20:20 + N]
            rd.copy_(res)
        yb = rnd(B, T, N + 12, seed=33).to(DEV)
        yd = yb[:, :, 4:4 + N]
        if y0 is not None:
            yd.copy_(y0)
        outside = torch.cat([yb[:, :, :4], yb[:, :, 4 + N:]], dim=2).clone()
    elif y0 is not None:
        yd = yd.clone()
    got = ops.conv1d(xd, w.to(DEV), bias.to(DEV), dilation=dil, pad_left=pad, in_act=in_act, in_slope=slope, out_act=out_act,
                     out_slope=0.1, res=rd, alpha=alpha, out=yd, accumulate=acc, row_lens=dv(lens), backend=1)
    torch.cuda.synchronize()
    if opts.get("strided"):
        assert torch.equal(torch.cat([yb[:, :, :4], yb[:, :, 4 + N:]], dim=2), outside)
    d = lambda t: None if t is None else t.double()
    want = E.conv1d(x.double(), w.double(), bias.double(), dil, pad, in_act, slope, out_act, 0.1, d(res), alpha, d(y0), lens)
    scale = conv_scale(x, w, bias, dil, pad, in_act, slope, res, alpha, y0, lens)
    err = normalised_err(got.cpu(), want, scale)
    tile = simt_plan(B, T, Cin, N, taps, torch.cuda.get_device_properties(0).multi_processor_count)
    parity_log("test_conv1d", case=str(case[:9]), tile=str(tile), err=err, bar=CONV_EXACT_C)
    assert err <= CONV_EXACT_C, (err, tile)


# Ragged batches (fs2_conv1d_args::x_lens): utterance b is computed on its first n_b = min(x_lens[b] * lens_scale, T) rows as if alone.
# Row counts 0, 1, BM - 1, BM, BM + 1 and T (and a length past T) for both row tiles.
RAGGED_CONV_CASES = [
    # B, T, Cin, N, taps, dil, pad, in_act, out_act, lens_scale, x_lens
    (6, 300, 64, 48, 5, 2, 4, 3, 3, 1, (0, 1, 63, 64, 65, 300)),                            # BM = 64
    (6, 12000, 32, 64, 7, 1, 3, 3, 0, 1, (12000, 127, 128, 129, 1, 0)),                     # BM = 128
    (6, 2400, 64, 96, 3, 1, 1, 0, 1, 8, (0, 1, 8, 16, 17, 300)),                             # lens_scale 8: rows 0, 8, 64, 128, 136, T
    (4, 17000, 16, 32, 11, 5, 25, 3, 3, 8, (2125, 16, 17, 9000)),                            # 9000 * 8 > T: clamped
]


@pytest.mark.parametrize("case", RAGGED_CONV_CASES)
def test_conv1d_ragged(case, parity_log):
    """The exact kernel on a ragged batch: each utterance's rows < n_b against fp64 of that utterance alone (T = n_b), with the rows
    at and past n_b of x and of the residual poisoned with NaN."""
    B, T, Cin, N, taps, dil, pad, in_act, out_act, scale_, xl = case
    x = rnd(B, T, Cin, seed=1)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    res = rnd(B, T, N, seed=4)
    n = [min(max(l * scale_, 0), T) for l in xl]
    for b in range(B):
        x[b, n[b]:] = float("nan"); res[b, n[b]:] = float("nan")
    got = ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), dilation=dil, pad_left=pad, in_act=in_act, in_slope=0.1, out_act=out_act,
                     out_slope=0.1, res=res.to(DEV), backend=1, x_lens=torch.tensor(xl, dtype=torch.int32, device=DEV),
                     lens_scale=scale_).cpu()
    errs = []
    for b in range(B):
        if n[b] == 0:
            continue
        xb, rb = x[b:b + 1, :n[b]], res[b:b + 1, :n[b]]
        want = E.conv1d(xb.double(), w.double(), bias.double(), dil, pad, in_act, 0.1, out_act, 0.1, rb.double())
        errs.append(normalised_err(got[b:b + 1, :n[b]], want, conv_scale(xb, w, bias, dil, pad, in_act, 0.1, rb, 1.0, None, None)))
    tile = simt_plan(B, T, Cin, N, taps, torch.cuda.get_device_properties(0).multi_processor_count)
    parity_log("test_conv1d_ragged", case=str(case), tile=str(tile), err=max(errs), bar=CONV_EXACT_C)
    assert max(errs) <= CONV_EXACT_C, (errs, tile)


def _lens(B, T, spec):
    """Per-utterance row counts of a case table entry: False = none, True = T - 7 (b + 1), or the lengths themselves."""
    if spec is False:
        return None
    if spec is True:
        return torch.tensor([max(1, T - 7 * (i + 1)) for i in range(B)], dtype=torch.int32)
    assert len(spec) == B
    return torch.tensor(spec, dtype=torch.int32)


def _ref_utts(B):
    """Utterances compared with the fp64 reference: all of a small batch, the first and the last of a large one.  The others are checked
    bit for bit against the same utterance run alone (the *_per_utterance_independence tests), which costs no CPU reference."""
    return list(range(B)) if B <= 3 else [0, B - 1]


def _conv_case(case):
    B, T, Cin, N, taps, dil, pad, in_act, out_act, use_res, alpha, acc, lens_spec = case
    x = rnd(B, T, Cin, seed=1)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    res = rnd(B, T, N, seed=4) if use_res else None
    y0 = rnd(B, T, N, seed=5) if acc else None
    return x, w, bias, res, y0, _lens(B, T, lens_spec)


def _sel(t, u):
    return None if t is None else t[u]


def tc_bars(got, u, x, w, bias, fmt, dil, pad, in_act, in_slope, out_act, res, alpha, y0, lens, seg_cin=None):
    """The two per-element bars of the tensor-core kernels (tests/emul_cabi.py::tc_errors) on the utterances u of a batched result:
    (a) against the rounded-operand contract, (b) against the unrounded fp64 conv; each normalised error must stay <= E.TC_ACC_C."""
    y_c, y64, S, R = E.tc_contract(x[u], w, bias, fmt, dil, pad, in_act, in_slope, out_act, 0.1, _sel(res, u), alpha, _sel(y0, u),
                                   _sel(lens, u), seg_cin=seg_cin)
    return E.tc_errors(got.cpu()[u], y_c, y64, S, R)


def _tc_call(case, x, w, bias, res, y0, lens, w_tc, variant):
    """fs2_conv1d on the tensor cores (backend = 2) for the case's epilogue settings; x, res, y0 and lens are CPU tensors."""
    _, _, _, _, _, dil, pad, in_act, out_act, _, alpha, acc, _ = case
    dv = lambda t: None if t is None else t.to(DEV)
    return ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), dilation=dil, pad_left=pad, in_act=in_act, in_slope=0.1, out_act=out_act,
                      out_slope=0.1, res=dv(res), alpha=alpha, out=y0.to(DEV).clone() if acc else None, accumulate=acc,
                      row_lens=dv(lens), w_tc=w_tc.to(DEV), backend=2, tc_variant=variant)


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
    # every work-item width the dispatcher instantiates (split3 NB / f8 NB): N = 16 -> 16 / 16, 48 -> 48 / 48, 192 -> 96 / 64
    (2, 300, 32, 16, 3, 1, 1, 3, 0, True, 1.0, False, False),
    (2, 260, 64, 48, 5, 2, 4, 3, 3, False, 1.0, False, True),
    (2, 390, 128, 192, 3, 1, 1, 0, 1, True, 0.5, True, False),
    # the slab's halo at its limit, (taps - 1) * dilation = 256 (every row of the transform warps' register ring), centred and
    # off-centre zero padding on multi-tile inputs
    (2, 700, 32, 64, 2, 256, 0, 0, 0, False, 1.0, False, False),
    (2, 700, 32, 64, 3, 128, 256, 3, 0, True, 1.0, False, False),
    (1, 1000, 16, 32, 3, 128, 128, 0, 0, False, 1.0, False, False),
]

# Shipped layer shapes at sizes where the persistent grid (min(work items, SMs)) gives every CTA of a 132-SM H100 at least two work
# items in both tile formats: the slab ring, the mbarrier phases and the producer's item walk carry over between items, and T % 128 != 0
# with ragged lengths makes consecutive items of one CTA straddle utterances and alternate interior / bounds-checked slabs.
# tests/test_abi.py checks the item counts against fs2_conv_tc_plan.
TC_PERSISTENT_CASES = [
    (6, 1012, 256, 1024, 9, 1, 4, 0, 1, False, 1.0, False, (1012, 873, 1012, 640, 955, 401)),   # decoder conv-FFN w_1 + ReLU
    (8, 2100, 1024, 256, 1, 1, 0, 0, 0, True, 1.0, False, (2100, 1999, 1500, 2100, 7, 1300, 2051, 650)),   # w_2 + residual
    (8, 1100, 512, 512, 5, 1, 2, 0, 2, False, 1.0, False, False),     # PostNet 512 -> 512 + tanh
    (8, 4200, 512, 80, 5, 1, 2, 0, 0, True, 1.0, False, (4200, 4100, 2500, 4199, 129, 3000, 4200, 1)),   # PostNet 512 -> 80 + mel
    (2, 40000, 64, 64, 11, 5, 25, 3, 3, False, 1.0, False, False),    # HiFi-GAN stage-3 ResBlock conv1 (lrelu in / out)
    (2, 33000, 64, 64, 7, 1, 3, 0, 0, True, 1.0 / 3, True, False),    # stage-3 conv2: residual, mean through alpha / accumulate
    (4, 3000, 64, 336, 3, 1, 1, 3, 0, False, 1.0, False, False),      # N = 336: NB = 112 (split3) / 48 (f8)
]
TC_CASES += TC_PERSISTENT_CASES


@pytest.mark.parametrize("case", TC_CASES)
def test_conv1d_tensor_core(case, parity_log):
    """fs2_conv1d through the three-MMA split (FS2 tile format 0) against its rounded-operand contract and against fp64 (tc_bars)."""
    dil, pad, in_act, out_act, alpha = case[5], case[6], case[7], case[8], case[10]
    x, w, bias, res, y0, lens = _conv_case(case)
    wtc = packing.pack_conv_tc(w)
    assert wtc is not None
    got = _tc_call(case, x, w, bias, res, y0, lens, wtc, 0)
    torch.cuda.synchronize()
    ea, eb = tc_bars(got, _ref_utts(x.shape[0]), x, w, bias, "split3", dil, pad, in_act, 0.1, out_act, res, alpha, y0, lens)
    parity_log("test_conv1d_tensor_core", case=str(case[:9]), err_contract=ea, err_fp64=eb, bar=E.TC_ACC_C)
    assert ea <= E.TC_ACC_C and eb <= E.TC_ACC_C, (ea, eb)


@pytest.mark.parametrize("case", TC_CASES)
def test_conv1d_tensor_core_f8_split(case, parity_log):
    """FS2_TC_VARIANT_F8 (fp16 main term + one E4M3 correction MMA): (a) the kernel computes exactly the rounded-operand products of
    its contract up to fp32 accumulation (so a wrong byte order / scale / K layout cannot hide), (b) against the unrounded fp64 conv it
    is within R, the E4M3 terms' stated precision (tc_bars)."""
    dil, pad, in_act, out_act, alpha = case[5], case[6], case[7], case[8], case[10]
    x, w, bias, res, y0, lens = _conv_case(case)
    got = _tc_call(case, x, w, bias, res, y0, lens, packing.pack_conv_tc(w, f8=True), 1)
    torch.cuda.synchronize()
    ea, eb = tc_bars(got, _ref_utts(x.shape[0]), x, w, bias, "f8", dil, pad, in_act, 0.1, out_act, res, alpha, y0, lens)
    parity_log("test_conv1d_tensor_core_f8_split", case=str(case[:9]), err_contract=ea, err_fp64=eb, bar=E.TC_ACC_C)
    assert ea <= E.TC_ACC_C and eb <= E.TC_ACC_C, (ea, eb)


SEG_CASES = [
    # B, T, Cin, N, taps, pad, in_act (0 none / 3 = lrelu slope 0 = ReLU), res, lens
    (2, 128, 256, 768, 1, 0, 0, False, False),      # encoder QKV projection
    (3, 100, 256, 1024, 9, 4, 0, False, False),     # conv-FFN w_1 (pre-activation output)
    (2, 128, 1024, 256, 1, 0, 3, True, True),       # conv-FFN w_2: ReLU on the input, residual, pad-row mask, 4 channel chunks
    (2, 300, 256, 256, 3, 1, 0, False, False),      # predictor conv, T > 256 (several tiles per utterance)
]
# Encoder layers at B = 16 with >= 2 work items per CTA on 132 SMs (at L = 128 QKV and w_1 give only 192 / 256 items): several 128-row
# tiles per utterance, ragged lengths; w_2 at a frame-level length (four 256-channel chunks per item).
SEG_PERSISTENT_CASES = [
    (16, 150, 256, 768, 1, 0, 0, False, (150, 149, 3, 128, 129, 150, 77, 100, 150, 1, 140, 131, 150, 64, 90, 127)),
    (16, 260, 256, 1024, 9, 4, 0, False, (260, 259, 3, 128, 129, 256, 77, 257, 150, 1, 240, 131, 260, 64, 90, 127)),
    (16, 600, 1024, 256, 1, 0, 3, True, (600, 513, 12, 600, 257, 384, 599, 100, 600, 450, 1, 333, 600, 578, 129, 200)),
]
SEG_CASES += SEG_PERSISTENT_CASES


def _seg_call(case, x, w, bias, res, lens, w_tc, backend=2):
    pad, in_act = case[5], case[6]
    dv = lambda t: None if t is None else t.to(DEV)
    return ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), pad_left=pad, in_act=in_act, in_slope=0.0, res=dv(res), row_lens=dv(lens),
                      w_tc=dv(w_tc), backend=backend, tc_variant=2 | 4 if w_tc is not None else 0)


def _seg_case(case):
    B, T, Cin, N, taps, pad, in_act, use_res, lens_spec = case
    x = rnd(B, T, Cin, seed=1)
    w = rnd(taps, Cin, N, seed=2, scale=(taps * Cin) ** -0.5)
    bias = rnd(N, seed=3, scale=0.1)
    res = rnd(B, T, N, seed=4) if use_res else None
    return x, w, bias, res, _lens(B, T, lens_spec)


@pytest.mark.parametrize("case", SEG_CASES)
def test_conv1d_tensor_core_k_segmented(case, parity_log):
    """FS2_TC_VARIANT_NB64 | FS2_TC_VARIANT_SEGMENTED: one launch whose work units are (tile, tap, 256-channel chunk) slices with fresh
    16-step accumulators, summed in fp32 through y, each slice scaled back with its own header.  tc_bars with the per-slice scales."""
    B, T, Cin, N, taps, pad, in_act = case[:7]
    x, w, bias, res, lens = _seg_case(case)
    wseg = packing.pack_conv_tc_segments(w)
    assert wseg is not None and wseg.numel() == taps * (Cin // 256) * (128 + 1024 * N)
    got = _seg_call(case, x, w, bias, res, lens, wseg)
    torch.cuda.synchronize()
    ea, eb = tc_bars(got, _ref_utts(B), x, w, bias, "split3", 1, pad, in_act, 0.0, 0, res, 1.0, None, lens, seg_cin=packing.SEG_CIN)
    parity_log("test_conv1d_tensor_core_k_segmented", case=str(case[:7]), err_contract=ea, err_fp64=eb, bar=E.TC_SEG_ACC_C)
    assert ea <= E.TC_SEG_ACC_C and eb <= E.TC_SEG_ACC_C, (ea, eb)


@pytest.mark.parametrize("fmt,case", [("split3", c) for c in TC_PERSISTENT_CASES] + [("f8", c) for c in TC_PERSISTENT_CASES]
                         + [("segmented", c) for c in SEG_PERSISTENT_CASES])
def test_conv1d_tensor_core_per_utterance_independence(fmt, case):
    """Each output element is produced by exactly one work item, whose arithmetic (K-block / tap order, epilogue) does not depend on
    the item's index or on what the CTA ran before it.  So every utterance of a batched call must equal, bit for bit, the same utterance
    run alone (B = 1, same T) -- a slab, mbarrier phase or weight stage carried over wrongly between one CTA's items breaks that."""
    if fmt == "segmented":
        x, w, bias, res, lens = _seg_case(case)
        wt = packing.pack_conv_tc_segments(w)
        run = lambda u: _seg_call(case, x[u], w, bias, _sel(res, u), _sel(lens, u), wt)
    else:
        x, w, bias, res, y0, lens = _conv_case(case)
        wt = packing.pack_conv_tc(w, f8=fmt == "f8")
        run = lambda u: _tc_call(case, x[u], w, bias, _sel(res, u), _sel(y0, u), _sel(lens, u), wt, 1 if fmt == "f8" else 0)
    got = run(slice(None))
    for b in range(x.shape[0]):
        alone = run(slice(b, b + 1))
        assert torch.equal(got[b:b + 1], alone), (b, (got[b:b + 1] - alone).abs().max().item())


@pytest.mark.parametrize("f8", [False, True])
def test_conv1d_tensor_core_strided_views(f8):
    """x a 32-byte-aligned channel slice of a wider buffer (row stride > Cin), res and y strided views of wider buffers, many work items
    per CTA: the result equals the same call on contiguous copies bit for bit (strides only move addresses), matches the contract, and
    the columns of the output buffer outside the view are left untouched."""
    B, T, Cin, N, taps, pad = 3, 12000, 64, 96, 5, 2
    case = (B, T, Cin, N, taps, 1, pad, 3, 0, True, 0.5, True, (12000, 11999, 4321))
    x, w, bias, res, y0, lens = _conv_case(case)
    xb = rnd(B, T, Cin + 24, seed=31).to(DEV)
    xs = xb[:, :, 8:8 + Cin]
    xs.copy_(x.to(DEV))
    assert xs.data_ptr() % 32 == 0 and xs.stride(1) == Cin + 24
    rb = rnd(B, T, N + 40, seed=32).to(DEV)
    rs = rb[:, :, 20:20 + N]
    rs.copy_(res.to(DEV))
    yb = rnd(B, T, N + 12, seed=33).to(DEV)
    ys = yb[:, :, 4:4 + N]
    ys.copy_(y0.to(DEV))
    outside = torch.cat([yb[:, :, :4], yb[:, :, 4 + N:]], dim=2).clone()
    wt = packing.pack_conv_tc(w, f8=f8).to(DEV)
    ops.conv1d(xs, w.to(DEV), bias.to(DEV), pad_left=pad, in_act=3, in_slope=0.1, res=rs, alpha=0.5, out=ys, accumulate=True,
               row_lens=lens.to(DEV), w_tc=wt, backend=2, tc_variant=int(f8))
    ref = _tc_call(case, x, w, bias, res, y0, lens, wt, int(f8))
    torch.cuda.synchronize()
    assert torch.equal(ys, ref)
    assert torch.equal(torch.cat([yb[:, :, :4], yb[:, :, 4 + N:]], dim=2), outside)
    ea, eb = tc_bars(ys, [0, 2], x, w, bias, "f8" if f8 else "split3", 1, pad, 3, 0.1, 0, res, 0.5, y0, lens)
    assert ea <= E.TC_ACC_C and eb <= E.TC_ACC_C, (ea, eb)


def test_conv1d_tensor_core_halo_limit():
    """(taps - 1) * dilation = 257 does not fit the slab the transform warps hold: FS2_CONV_TC refuses it, FS2_CONV_AUTO serves it with
    the exact fp32 kernel."""
    from fastspeech2_b200._lib import Fs2Error
    B, T, Cin, N = 2, 600, 32, 64
    x = rnd(B, T, Cin, seed=51)
    w = rnd(2, Cin, N, seed=52, scale=0.1)
    wt = packing.pack_conv_tc(w).to(DEV)
    with pytest.raises(Fs2Error):
        ops.conv1d(x.to(DEV), w.to(DEV), None, dilation=257, pad_left=128, w_tc=wt, backend=2)
    got = ops.conv1d(x.to(DEV), w.to(DEV), None, dilation=257, pad_left=128, w_tc=wt, backend=0)
    torch.cuda.synchronize()
    want = E.conv1d(x.double(), w.double(), None, 257, 128)
    assert (got.cpu().double() - want).abs().max().item() < 5e-6


RESSTACK_CASES = [
    # B, N, C, kernels, dilations
    (1, 700, 32, (3, 7, 11), ((1, 3, 5),) * 3),       # two work items, ragged second tile
    (2, 392 * 2, 32, (3, 7, 11), ((1, 3, 5),) * 3),   # exact multiple of the tile
    (2, 100, 32, (3, 7, 11), ((1, 3, 5),) * 3),       # utterance shorter than the halo-extended slab
    (2, 900, 64, (3, 7, 11), ((1, 3, 5),) * 3),       # 64 channels: three 128-row tiles per slab
    (1, 264, 64, (3, 7, 11), ((1, 3, 5),) * 3),       # 64 channels: two tiles, ragged second one
    (3, 50, 64, (3, 5), ((1, 2), (2, 6))),            # other kernel sets / dilation lists
    # the shipped group at one sample and at one tile +- 1 row (fs2_resstack_plan: TILE = 392 at C = 32, 136 at C = 64)
    (2, 1, 32, (3, 7, 11), ((1, 3, 5),) * 3),
    (2, 391, 32, (3, 7, 11), ((1, 3, 5),) * 3),
    (2, 393, 32, (3, 7, 11), ((1, 3, 5),) * 3),
    (2, 1, 64, (3, 7, 11), ((1, 3, 5),) * 3),
    (2, 135, 64, (3, 7, 11), ((1, 3, 5),) * 3),
    (1, 136, 64, (3, 7, 11), ((1, 3, 5),) * 3),
    (2, 137, 64, (3, 7, 11), ((1, 3, 5),) * 3),
]
RESSTACK_TILE = {32: 392, 64: 136}      # output rows per work item of the shipped group (tests/test_abi.py checks it against the plan)



def _resstack_case(case):
    """Input and per-layer weights of a RESSTACK_CASES entry: x [B,N,C], and per (kernel size j, dilation d) the conv weights in the
    fs2_conv1d layout [k][C][C] and their biases."""
    B, N, C, kernels, dils = case
    x = rnd(B, N, C, seed=21)
    w1, b1, w2, b2 = [], [], [], []
    for j, k in enumerate(kernels):
        w1.append([]); b1.append([]); w2.append([]); b2.append([])
        for d in range(len(dils[j])):
            w1[j].append(packing.conv_w(rnd(C, C, k, seed=100 + 10 * j + d, scale=0.6 * (C * k) ** -0.5)))      # from [out, in, k]
            w2[j].append(packing.conv_w(rnd(C, C, k, seed=200 + 10 * j + d, scale=0.6 * (C * k) ** -0.5)))
            b1[j].append(rnd(C, seed=300 + 10 * j + d, scale=0.05)); b2[j].append(rnd(C, seed=400 + 10 * j + d, scale=0.05))
    return x, w1, b1, w2, b2


@pytest.mark.parametrize("case", RESSTACK_CASES)
def test_resstack_fused(case, parity_log):
    """fs2_resstack (one persistent kernel for a whole multi-receptive-field ResBlock group, intermediates on chip, halo recompute)
    (b) against an fp64 evaluation of hifigan/models.py:96-103,:154-160 within R, the f16 + f8 format's bound carried through the
    group, and (a) against the same group built from per-layer tensor-core convs on the same tiles, which leaves only accumulation order;
    both per element, scaled by S carried through the group (tests/test_gpu_tc_precision.py::resstack_check)."""
    from tests.test_gpu_tc_precision import resstack_check
    B, N, C, kernels, dils = case
    x, w1, b1, w2, b2 = _resstack_case(case)
    resstack_check("test_resstack_fused", x, kernels, dils, w1, b1, w2, b2, parity_log, case=str(case))


SINGLE_PAIR_CASES = [
    # C, k, dilations, N
    (64, 3, (5,), 1000), (64, 7, (3,), 1000), (32, 3, (1,), 1000), (64, 11, (5,), 777), (32, 11, (5,), 1500),
    (32, 7, (3,), 900), (64, 3, (1, 3, 5), 1234), (64, 3, (1,), 21000), (32, 7, (1,), 40000), (64, 5, (2,), 40),
    # every tap reaching exactly 32 rows outside the tile ((k - 1) * dil / 2 = 32, the limit of the fs2_resstack contract)
    (32, 3, (32,), 3000), (32, 5, (16,), 1000), (32, 9, (8,), 1000),
    (64, 3, (32,), 3000), (64, 5, (16,), 1000), (64, 9, (8,), 1000),
]


@pytest.mark.parametrize("C,k,dils,N", SINGLE_PAIR_CASES)
def test_resstack_single_pair_accumulate(C, k, dils, N):
    """The single-kernel-size mode of fs2_resstack (n_kernels = 1, alpha, accumulate): y += alpha * ResBlock_k,dils(x).  The long cases
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


CONV_TRANSPOSE_CASES = [
    # u, C_in, C_out, T
    (8, 64, 32, 37), (2, 64, 32, 130),
    (8, 512, 256, 300),       # HiFi-GAN stage 1: N = 1024 per phase group
    (2, 128, 64, 20000),      # stage 3: >= 2 work items per CTA of a 132-SM grid in both tile formats
]


def _conv_transpose_check(u, cin, cout, T, fmt, parity_log):
    """lrelu + ConvTranspose1d as the vocoder runs it: two 2-tap phase-group convs whose outputs interleave in the rows of one
    [B, T, u*C_out] buffer (y_row_stride = u*C_out).  Against fp64 torch conv_transpose1d; f8 also against its rounded-operand
    contract."""
    w = rnd(cin, cout, 2 * u, seed=7, scale=0.1)
    x = rnd(2, T, cin, seed=8)
    bias = rnd(cout, seed=9, scale=0.1)
    want = torch.nn.functional.conv_transpose1d(torch.nn.functional.leaky_relu(x.double(), 0.1).transpose(1, 2), w.double(), bias.double(),
                                                stride=u, padding=u // 2).transpose(1, 2)
    wa, wb = packing.split_conv_transpose(w, u)
    half = u // 2
    out = torch.empty(2, T, u * cout, device=DEV)
    bt = bias.repeat(u)
    xd = x.to(DEV)
    kw = {} if fmt == "fp32" else dict(backend=2, tc_variant=int(fmt == "f8"))
    tile = lambda w_: None if fmt == "fp32" else packing.pack_conv_tc(w_, f8=fmt == "f8").to(DEV)
    ops.conv1d(xd, wa.to(DEV), bt[: half * cout].to(DEV), pad_left=1, in_act=3, in_slope=0.1, out=out[:, :, : half * cout], w_tc=tile(wa), **kw)
    ops.conv1d(xd, wb.to(DEV), bt[half * cout:].to(DEV), pad_left=0, in_act=3, in_slope=0.1, out=out[:, :, half * cout:], w_tc=tile(wb), **kw)
    torch.cuda.synchronize()
    err = (out.cpu().double().reshape(2, T * u, cout) - want).abs().max().item()
    if fmt == "fp32":
        parity_log("test_conv1d_strided_output_conv_transpose", case=f"{fmt} u={u} {cin}->{cout} T={T}", err=err, bar=2e-5)
        assert err < 2e-5, err
        return
    # the tensor-core phase groups: tc_bars on each group's columns, and the interleaved rows against torch's conv_transpose1d
    both = [0, 1]
    ea, eb = tc_bars(out[:, :, : half * cout], both, x, wa, bt[: half * cout], fmt, 1, 1, 3, 0.1, 0, None, 1.0, None, None)
    ea2, eb2 = tc_bars(out[:, :, half * cout:], both, x, wb, bt[half * cout:], fmt, 1, 0, 3, 0.1, 0, None, 1.0, None, None)
    ea, eb = max(ea, ea2), max(eb, eb2)
    cat = torch.cat([E.conv1d(x.double(), wa.double(), bt[: half * cout].double(), 1, 1, 3, 0.1),
                     E.conv1d(x.double(), wb.double(), bt[half * cout:].double(), 1, 0, 3, 0.1)], dim=2).reshape(2, T * u, cout)
    assert (cat - want).abs().max().item() < 1e-12            # the phase split itself is exact
    parity_log("test_conv1d_strided_output_conv_transpose", case=f"{fmt} u={u} {cin}->{cout} T={T}", err_contract=ea, err_fp64=eb,
               bar=E.TC_ACC_C)
    assert ea <= E.TC_ACC_C and eb <= E.TC_ACC_C, (ea, eb)


def test_conv1d_strided_output_conv_transpose(parity_log):
    """The phase-group ConvTranspose on the fp32 CUDA-core kernel."""
    for u, cin, cout, T in CONV_TRANSPOSE_CASES:
        _conv_transpose_check(u, cin, cout, T, "fp32", parity_log)


@pytest.mark.parametrize("fmt", ["split3", "f8"])
@pytest.mark.parametrize("u,cin,cout,T", CONV_TRANSPOSE_CASES)
def test_conv1d_tensor_core_strided_output_conv_transpose(u, cin, cout, T, fmt, parity_log):
    """The phase-group ConvTranspose on the tensor cores, in both tile formats (the vocoder's default for stages 1-4 is f8)."""
    _conv_transpose_check(u, cin, cout, T, fmt, parity_log)


def test_conv1d_rejects_bad_shapes():
    from fastspeech2_b200._lib import Fs2Error
    x = torch.zeros(1, 8, 24, device=DEV)          # Cin % 16 != 0
    w = torch.zeros(1, 24, 16, device=DEV)
    with pytest.raises(Fs2Error):
        ops.conv1d(x, w)


# |y - y64| <= LN_C * 2^-24 * (|gamma| max|x| / sqrt(var + eps) + |beta|) per element (ln_scale).  Largest value measured on an
# H100 80GB HBM3 (700 W power limit): 3.2, so the bar leaves 5x headroom.
LN_C = 16.0


# Constant rows: every one but 0.1 has exact fp32 partial sums at any C <= 1024 in any order.
LN_CONSTANTS = (0.0, 1.0, -7.5, 0.1, 1234.5, -3.0e4)


def layernorm_rows(C, seed=1):
    """[3, 50, C]: N(0.5, 3) rows, then rows whose |mean| / std is 1e2 .. 1e4 (where E[x^2] - E[x]^2 in fp32 cancels catastrophically)
    and constant rows (output = beta)."""
    x = rnd(3, 50, C, seed=seed, scale=3.0) + 0.5
    for i, (ratio, sign) in enumerate(((1e2, 1), (3e2, -1), (1e3, 1), (3e3, -1), (1e4, 1), (1e4, -1))):
        std = 0.25 * (i + 1)
        x[0, 2 + i] = sign * ratio * std + std * rnd(C, seed=seed + 10 + i)
    for i, c in enumerate(LN_CONSTANTS):
        x[0, 10 + i] = c
        x[1, 5 + i] = c
    return x


def ln_scale(x, gamma, beta):
    xd = x.double()
    var = xd.var(-1, unbiased=False, keepdim=True)
    return gamma.double().abs() * xd.abs().amax(-1, keepdim=True) / (var + 1e-5).sqrt() + beta.double().abs()


@pytest.mark.parametrize("C", [256, 512, 1024, 80])
def test_layernorm(C, parity_log):
    """fs2_layernorm against fp64, with rows where a one-pass variance fails and constant rows, within a bar relative to the row's
    max |x| / std."""
    x = layernorm_rows(C)
    gm, bt = 1 + rnd(C, seed=2, scale=0.1), rnd(C, seed=3, scale=0.1)
    lens = torch.tensor([50, 13, 1], dtype=torch.int32)
    errs = []
    for ln_ in (None, lens):
        # pre_relu: the predictors' conv -> ReLU -> LayerNorm with the ReLU left to this op
        for pre_relu in (False, True):
            xr = torch.relu(x) if pre_relu else x
            want = E.layernorm(xr.double(), gm.double(), bt.double(), ln_)
            got = ops.layernorm(x.to(DEV), gm.to(DEV), bt.to(DEV), None if ln_ is None else ln_.to(DEV), pre_relu=pre_relu).cpu()
            scale = ln_scale(xr, gm, bt)
            if ln_ is not None:
                scale = scale.masked_fill((torch.arange(50)[None, :] >= ln_[:, None])[..., None], 0.0)
            errs.append(normalised_err(got, want, scale))
            # constant rows give beta.  With C a power of two the mean of an exactly summable row is exact, x - mean = 0 and y = beta bit for
            # bit.  Otherwise the mean's rounding leaves up to an ulp of x, which 1 / sqrt(eps) amplifies: only the (loose) bar applies.
            for i, c in enumerate(LN_CONSTANTS):
                if C & (C - 1) == 0 and c != 0.1:
                    assert torch.equal(got[0, 10 + i], bt), c
                else:
                    assert ((got[0, 10 + i] - bt).abs() <= LN_C * U24 * scale[0, 10 + i]).all(), c
    parity_log("test_layernorm", case=f"C={C}", err=max(errs), bar=LN_C)
    assert max(errs) <= LN_C, errs


def test_wav_to_int16():
    """fs2_wav_to_int16 against numpy's astype("int16") (truncation toward zero) on in-range samples; the documented clamp at and
    beyond +-1.0 * 32768; lengths None / 0 / negative / > N; N % 8 != 0 with a row-strided wav whose rows are not 16-byte aligned (the
    scalar load / store branch)."""
    import numpy as np
    B, N = 4, 1003
    buf = torch.rand(B, N + 5, generator=g(61)) * 1.9998 - 0.9999          # in (-1, 1)
    wav = buf[:, :N]
    assert wav.stride(0) == N + 5
    want = (wav.numpy() * np.float32(32768.0)).astype("int16")
    got = ops.wav_to_int16(wav.to(DEV)).cpu().numpy()
    assert np.array_equal(got, want)
    got = ops.wav_to_int16(buf.to(DEV)[:, :N]).cpu().numpy()                 # the same rows read through a strided device view
    assert np.array_equal(got, want)
    lens = torch.tensor([N + 100, 0, -5, 517])
    got = ops.wav_to_int16(buf.to(DEV)[:, :N], lens).cpu().numpy()
    keep = np.arange(N)[None, :] < lens.clamp(0, N).numpy()[:, None]
    assert np.array_equal(got, np.where(keep, want, 0))
    edge = torch.tensor([[1.0, -1.0, 1.5, -1.5, 1e9, -1e9, float("inf"), -float("inf"), 0.99999, -0.99999, 32767 / 32768, -32767 / 32768]])
    got = ops.wav_to_int16(edge.to(DEV)).cpu().tolist()[0]
    assert got == [32767, -32768, 32767, -32768, 32767, -32768, 32767, -32768, 32767, -32767, 32767, -32767]


def test_add_positions():
    """fs2_add_positions: x[b,t,:] += pos[t,:], one fp32 add per element, so bit for bit torch's x + pos[:T]."""
    x = rnd(3, 517, 256, seed=71)
    pos = rnd(1001, 256, seed=72)
    got = ops.add_positions_(x.to(DEV), pos.to(DEV))
    assert torch.equal(got.cpu(), x + pos[:517])


ATT_ADV_CASES = [
    ("random", 256, [256, 200, 129, 128, 127, 77, 65, 64, 63, 40, 17, 9, 3, 1, 256, 250] * 4),     # encoder shape B = 64 (configs[3]-like)
    ("random", 300, EDGE_LENS),
    ("last_tile_max", 300, EDGE_LENS),
    ("masked_max", 300, EDGE_LENS),
    ("range80", 300, EDGE_LENS),
    ("tied", 300, EDGE_LENS),
    ("last_tile_max", 1012, [1012, 1000, 640]),
]
ATT_DECODER_CASES = [("random", 1012, [1012, 998]), ("random", 2000, [2000, 1999]), ("last_tile_max", 4200, [4200, 4097])]


def _attention_check(kind, T, lens, backend, parity_log):
    qkv = attention_qkv(kind, lens, T)
    kl = torch.tensor(lens, dtype=torch.int32)
    got = ops.attention(qkv.to(DEV), 2, kl.to(DEV), backend=backend).cpu()
    assert torch.isfinite(got).all()
    for b, n in enumerate(lens):                         # padded query rows are exact zeros
        assert (got[b, max(n, 0):] == 0).all()
    err = 0.0
    for b in range(len(lens)):
        want = E.attention(qkv[b:b + 1].double(), 2, kl[b:b + 1])
        err = max(err, attention_normalised_err(got[b:b + 1], want, attention_bar_scale(qkv[b:b + 1], kl[b:b + 1])))
    top_err = 0.0
    if kind == "range80":                                # O is the argmax key's v itself, to fp32 accuracy
        v = qkv[..., 512:]
        for b, n in enumerate(lens):
            n = min(max(n, 0), T)
            if n:
                top = v[b, n // 2]
                top_err = max(top_err, ((got[b, :n] - top).abs().max() / (U24 * top.abs().max())).item())
    parity_log("test_attention", case=f"backend={backend} {kind} B={len(lens)} T={T}", err=err, bar=ATT_EXACT_C[backend], top_err=top_err)
    assert err <= ATT_EXACT_C[backend] and top_err <= ATT_EXACT_C[backend], (kind, T, err, top_err)


@pytest.mark.parametrize("backend", [0, 2])
@pytest.mark.parametrize("kind,T,lens", ATT_ADV_CASES)
def test_attention_adversarial_scores(kind, T, lens, backend, parity_log):
    """fs2_attention, both backends, against fp64 E.attention with a per-row bar that grows with the score range: lengths 0, 1,
    64k +- 1, past T and negative; the row max in the last key tile; masked keys holding the largest scores; a +-80-nat range; ties."""
    _attention_check(kind, T, lens, backend, parity_log)


@pytest.mark.parametrize("kind,T,lens", ATT_DECODER_CASES)
def test_attention_exact_decoder_lengths(kind, T, lens, parity_log):
    """The exact kernel (backend 0) at decoder lengths: it runs the whole decoder under tc_mask = 0."""
    _attention_check(kind, T, lens, 0, parity_log)


@pytest.mark.parametrize("T,lens", [(130, [130, 64, 1]), (64, [64, 64, 33]), (257, [257, 200, 65])])
def test_attention(T, lens):
    qkv = rnd(3, T, 768, seed=1)
    kl = torch.tensor(lens, dtype=torch.int32)
    want = E.attention(qkv, 2, kl)
    got = ops.attention(qkv.to(DEV), 2, kl.to(DEV))
    torch.cuda.synchronize()
    assert (got.cpu() - want).abs().max() < 5e-6


# work items of the fused kernel: B * heads * ceil(T / 128).  The benchmark batch (B = 16, T = 1012) has 256: some CTAs of a 132-SM
# grid take two; at T = 1100 every CTA does (288).
ATT_BATCHED_CASES = [
    (1012, [1012, 998, 1012, 877, 640, 1012, 1, 513, 1011, 129, 128, 900, 1012, 64, 777, 300]),
    (1100, [1100, 1, 1099, 1024, 1025, 77, 1100, 640, 128, 129, 1000, 1100, 5, 999, 256, 513]),
]


@pytest.mark.parametrize("T,lens", [(128, [128, 5, 77]), (300, [300, 129, 1]), (1017, [1017, 777, 513]), (1100, [1100, 64, 1037]),
                                    (4200, [4200, 4097, 9])] + ATT_BATCHED_CASES + [(1000, [1000, 777, 513])])
def test_attention_fused_kernel(T, lens, parity_log):
    """fs2_attention backend 2: QK^T, softmax and PV in ONE tensor-core kernel (scores stay in registers; two-pass softmax; no length
    limit) against an fp64 evaluation of transformer/Modules.py:14-25 with the key mask of Models.py:79: fp32-class accuracy."""
    qkv = rnd(len(lens), T, 768, seed=3)
    kl = torch.tensor(lens, dtype=torch.int32)
    u = _ref_utts(len(lens))
    want = E.attention(qkv[u].double(), 2, kl[u])
    got = ops.attention(qkv.to(DEV), 2, kl.to(DEV), backend=2)
    torch.cuda.synchronize()
    assert torch.isfinite(got).all()
    err = (got.cpu()[u].double() - want).abs().max().item()
    parity_log("test_attention_fused_kernel", case=f"B={len(lens)} T={T}", err=err, bar=2e-5)
    assert err < 2e-5, err
    # padded query rows are written as exact zeros (contract of fs2_attention)
    for b, n in enumerate(lens):
        assert (got[b, n:] == 0).all()


@pytest.mark.parametrize("T,lens", ATT_BATCHED_CASES)
def test_attention_fused_per_utterance_independence(T, lens):
    """One work item = one (utterance, head, 128-query tile) with the whole softmax over that utterance's keys: every utterance of a
    batched call equals, bit for bit, the same utterance run alone at the same T."""
    qkv = rnd(len(lens), T, 768, seed=3).to(DEV)
    kl = torch.tensor(lens, dtype=torch.int32).to(DEV)
    got = ops.attention(qkv, 2, kl, backend=2)
    for b in range(len(lens)):
        alone = ops.attention(qkv[b:b + 1].contiguous(), 2, kl[b:b + 1].contiguous(), backend=2)
        assert torch.equal(got[b:b + 1], alone), (b, (got[b:b + 1] - alone).abs().max().item())


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
    """torch.bucketize(right=False): a value equal to an edge goes to that edge's index, NaN past the last edge (ATen's search)."""
    bins = torch.linspace(-1.0, 1.0, 255)
    vals = torch.cat([bins[[0, 1, 100, 254]], torch.tensor([-5.0, 5.0, 0.0, -0.0, float("nan"), float("inf"), float("-inf")]),
                      torch.nextafter(bins[[0, 127, 254]], torch.tensor(2.0)), torch.nextafter(bins[[0, 127, 254]], torch.tensor(-2.0))])
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
    wd, wcum, wlen, _ = E.durations(logd, False, d_control)
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
    _, wcum2, wlen2, _ = E.durations(tgt, True, 1.0)
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
