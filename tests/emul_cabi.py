"""CPU emulation of the C-ABI operator semantics and of model.cu's orchestration (TEST INFRASTRUCTURE).

It consumes the SAME packed weights the CUDA path gets (fastspeech2_b200.packing) and follows the launch sequence of
fastspeech2_b200/csrc/model.cu op for op, with every op implemented from the contract written in include/fs2b200.h.
Comparing it with the oracle on CPU validates the decomposition (weight layouts, BatchNorm / weight-norm folds,
ConvTranspose phase split, duration prefix sums + upper_bound gather, padding rules) without a GPU; the `-m gpu`
tests then check that the kernels implement those op contracts.
"""
import math

import torch

ACT_NONE, ACT_RELU, ACT_TANH, ACT_LRELU = 0, 1, 2, 3


def _act(v, act, slope):
    if act == ACT_RELU:
        return torch.relu(v)
    if act == ACT_TANH:
        return torch.tanh(v)
    if act == ACT_LRELU:
        return torch.where(v > 0, v, v * slope)
    return v


def conv1d(x, w, bias, dilation=1, pad_left=0, in_act=ACT_NONE, in_slope=0.0, out_act=ACT_NONE, out_slope=0.0,
           res=None, alpha=1.0, y_prev=None, row_lens=None):
    """fs2_conv1d contract.  x [B,T,Cin], w [taps][Cin][N] -> [B,T,N]."""
    B, T, _ = x.shape
    taps, _, N = w.shape
    xa = _act(x, in_act, in_slope)
    acc = torch.zeros(B, T, N, dtype=x.dtype)
    for j in range(taps):
        shift = j * dilation - pad_left
        lo, hi = max(0, -shift), min(T, T - shift)
        if hi > lo:
            acc[:, lo:hi] += xa[:, lo + shift:hi + shift] @ w[j]
    return conv1d_epilogue(acc, bias, out_act, out_slope, res, alpha, y_prev, row_lens)


def conv1d_epilogue(acc, bias, out_act=ACT_NONE, out_slope=0.0, res=None, alpha=1.0, y_prev=None, row_lens=None):
    """Everything fs2_conv1d does after the tap / channel sums (bias, activation, residual, alpha, accumulate, pad-row mask)."""
    T = acc.shape[1]
    if bias is not None:
        acc = acc + bias
    v = _act(acc, out_act, out_slope)
    if res is not None:
        v = v + res
    v = v * alpha
    if y_prev is not None:
        v = v + y_prev
    if row_lens is not None:
        v = v.masked_fill((torch.arange(T)[None, :] >= row_lens[:, None])[..., None], 0.0)
    return v


def f8_operands(x, w, in_act=ACT_NONE, in_slope=0.0):
    """The operands the f16 + f8 tensor-core kernel multiplies, evaluated exactly: returns (a_hi, w_hi, a_lo8, w_hi8, a_hi8, w_lo8, scale)
    in fp64 so that  y*scale = a_hi.w_hi + a_lo8.w_hi8 + a_hi8.w_lo8  (tc_pipeline.cuh::split_f8x2, packing.pack_conv_tc)."""
    from fastspeech2_b200 import packing
    e4 = lambda t: t.float().clamp(-448, 448).to(torch.float8_e4m3fn).double()
    a = x.float()
    if in_act == ACT_LRELU:
        a = torch.maximum(a, a * in_slope)
    ah = a.half().float()
    al = a - ah
    hi, _, s = packing.split_fp16(w)
    wl = w.float() * s - hi.float()
    return (ah.double(), hi.double(), e4(al * 4096.0) / 4096.0, e4(hi.float() * 2.0 ** -12) * 4096.0, e4(ah), e4(wl), s)


def conv1d_f8(x, w, bias, dilation=1, pad_left=0, in_act=ACT_NONE, in_slope=0.0, out_act=ACT_NONE, out_slope=0.0,
              res=None, alpha=1.0, y_prev=None, row_lens=None, fp16_only=False):
    """fs2_conv1d with the f16 + f8 tile format (FS2_TC_VARIANT_F8) in fp64 on the rounded operands: what the kernel computes up to
    its fp32 accumulation.  x is rounded to fp32 first, as the kernel reads it.  fp16_only: drop the E4M3 correction term (a
    single-pass fp16 convolution), the error a kernel that lost the correction would make."""
    ah, wh, al8, wh8, ah8, wl8, s = f8_operands(x, w, in_act, in_slope)
    lin = lambda a_, w_: conv1d(a_, w_, None, dilation, pad_left)
    pre = lin(ah, wh) if fp16_only else lin(ah, wh) + lin(al8, wh8) + lin(ah8, wl8)
    d = lambda t: None if t is None else t.double()
    return conv1d_epilogue(pre / s, d(bias), out_act, out_slope, d(res), alpha, d(y_prev), row_lens)


# ------------------------------------------------------------------ tensor-core operand formats, bit for bit, and their error bounds
#
# Both formats multiply rounded operands and accumulate in fp32; in fp64 the rounded products are exact, so the contract
#     y_c = epilogue( sum_terms conv(A, W) )
# is what the kernel computes up to its fp32 accumulation, and a list of (A, W) pairs describes every format:
#   split3 (format 0):  (a_hi, w_hi/s) + (a_lo, w_hi/s) + (a_hi, w_lo/s)                     hi = fp16(v), lo = fp16(v - hi)
#   f8     (format 1):  (a_hi, w_hi/s) + (e4(a_lo 2^12)/2^12, e4(w_hi 2^-12) 2^12/s) + (e4(a_hi), e4(w_lo)/s)   lo = v - hi exact
# with a = in_act(x) in fp32, w scaled by the layer's power of two s (fp16 and E4M3 keep their subnormals; both converts saturate).
# Two bars per output element (tc_errors): (a) |y - y_c| <= TC_ACC_C 2^-24 S and (b) |y - y64| <= TC_ACC_C 2^-24 S + R.  After the
# operand rounding all that is left is the tensor core's fp32 accumulation: each 16-deep K-step sums its products (an error of a few
# ulp of their absolute sum) and adds them to the accumulator with truncation (at most one ulp of the running sum).  So S = the
# contract on absolute products, plus the accumulator mass: the sum over K-steps, in the kernel's order, of |running sum| (fp64, on
# the contract's terms), plus the epilogue terms.  The mass follows how the accumulator actually grows: about n S / 2 for a sum of one
# sign over n K-steps, about sqrt(n) S for random signs, so the bar stays tight on long random-signed sums without failing long
# one-signed ones.  R = the format's stated precision (a_bounds / w_bounds) carried through the epilogue, against the unrounded y64.

U24 = 2.0 ** -24
# Largest normalised error measured over every tensor-core conv test (tests/test_gpu_tc_precision.py incl. the shipped checkpoints'
# layers, tests/test_gpu_ops.py) on an H100 80GB HBM3 at a 700 W power limit: 5.1 (split3, weight outliers, several work items per
# CTA; the shipped checkpoints' layers reach 4.4), so the bar leaves 3.2x.  Not more: tests/test_tc_precision_cpu.py checks that a
# kernel without its correction terms, or without its activation lo plane, exceeds it by 10x on every shape these tests run, and the
# longest shipped sums (HiFi-GAN stage-0 ResBlock convs, 176 K-steps) come within 1.02x of that.
TC_ACC_C = 16.0
# The same for the K-segmented path (16-step slices added into y in fp32 round-to-nearest): 1.04, measured likewise.
TC_SEG_ACC_C = 4.0
E4M3_MAX = 448.0


def weight_scale(w):
    """The per-layer power of two s of the tensor-core tiles: the largest 2^k with s max|w| <= 2^14 (1 for an all-zero or non-finite
    w), derived here from frexp rather than from packing.split_fp16, so that the packer is checked against an independent definition."""
    m = float(w.abs().max())
    if m == 0.0 or not math.isfinite(m):
        return 1.0
    f, e = math.frexp(m)                      # m = f 2^e, f in [0.5, 1)
    return 2.0 ** (14 - e + (1 if f == 0.5 else 0))


def _f16(t):
    """fp32 -> fp16 round-to-nearest, subnormals kept, saturating at +-65504 (cvt.rn.satfinite.f16x2.f32), as fp32."""
    return t.clamp(-65504.0, 65504.0).half().float()


def _e4(t):
    """fp32 -> E4M3 round-to-nearest, subnormals kept, saturating at +-448 (cvt.rn.satfinite.e4m3x2.f32), as fp64."""
    return t.float().clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).double()


def _e4_err(v):
    """Bound on |v - e4(v)| from the E4M3 definition: half an ulp of 3 mantissa bits (2^-4 |v|), half the subnormal spacing 2^-9,
    or the saturation loss |v| - 448; never more than |v| itself below the saturation."""
    v = v.double().abs()
    return torch.maximum(torch.maximum(v * 2.0 ** -4, v.clamp_max(2.0 ** -10)), v - E4M3_MAX)


def _split3_err(v):
    """Bound on |v - (hi + lo)| of the fp16 hi / lo split: 2^-11 relative in lo, so 2^-22 |v|, and half of fp16's subnormal spacing
    2^-24 where lo (or hi itself) is subnormal: the absolute floor 2^-25 that every |v| below about 2^-3 reaches.  Valid for |v| <= 65504."""
    v = v.double().abs()
    return torch.maximum(v * 2.0 ** -22, v.clamp_max(2.0 ** -25))


def act_operand(x, in_act=ACT_NONE, in_slope=0.0):
    """The fp32 activation the kernel splits: x read as fp32, leaky_relu as fmaxf(a, a * slope) (0 <= slope <= 1)."""
    a = x.float()
    if in_act == ACT_LRELU:
        a = torch.maximum(a, a * in_slope)
    elif in_act != ACT_NONE:
        raise ValueError("the tensor-core kernel takes no other input activation")
    return a


def a_planes(a, fmt):
    """Activation side of each term (same order as w_planes), fp64."""
    ah = _f16(a)
    if fmt == "split3":
        return [ah.double(), _f16(a - ah).double(), ah.double()]
    return [ah.double(), _e4((a - ah) * 4096.0) / 4096.0, _e4(ah)]


def a_bounds(a, fmt):
    """Activation side of each term of R (same order as w_bounds), fp64 and nonnegative."""
    ah = _f16(a)
    lo = (a - ah).double().abs()
    if fmt == "split3":
        e = _split3_err(a)
        return [lo + e, a.double().abs() + e, e]
    ea, eh = _e4_err((a - ah) * 4096.0) / 4096.0, _e4_err(ah)
    return [ea, lo + ea, eh, ah.double().abs() + eh, lo]


def _w_split(w, fmt):
    s = weight_scale(w)
    ws = w.float() * s
    wh = ws.half().float()
    return s, ws, wh


def w_planes(w, fmt):
    """Weight side of each term, with 1/s applied (exact: s is a power of two), fp64 [taps][Cin][N]."""
    s, ws, wh = _w_split(w, fmt)
    if fmt == "split3":
        return [wh.double() / s, wh.double() / s, _f16(ws - wh).double() / s]
    return [wh.double() / s, _e4(wh * 2.0 ** -12) * 4096.0 / s, _e4(ws - wh) / s]


def w_bounds(w, fmt):
    s, ws, wh = _w_split(w, fmt)
    lo = (ws - wh).double().abs()
    if fmt == "split3":
        e = _split3_err(ws)
        return [(lo + e) / s, e / s, ws.double().abs() / s]
    return [wh.double().abs() / s, _e4_err(wh * 2.0 ** -12) * 4096.0 / s, lo / s, _e4_err(ws - wh) / s, lo / s]


def _segmented(fn, w, seg_cin):
    """fn applied to every (tap, seg_cin-channel) slice of w on its own (the K-segmented tiles: one scale per slice), reassembled."""
    if seg_cin is None:
        return fn(w)
    taps, cin, _ = w.shape
    parts = [[fn(w[t:t + 1, c:c + seg_cin]) for c in range(0, cin, seg_cin)] for t in range(taps)]
    return [torch.cat([torch.cat([p[i] for p in row], dim=1) for row in parts], dim=0) for i in range(len(parts[0][0]))]


def _pairs(x, w, fmt, in_act, in_slope, seg_cin):
    a = act_operand(x, in_act, in_slope)
    fn_w = (lambda v: w_planes(v, fmt)), (lambda v: w_bounds(v, fmt))
    terms = list(zip(a_planes(a, fmt), _segmented(fn_w[0], w, seg_cin)))
    bound = list(zip(a_bounds(a, fmt), _segmented(fn_w[1], w, seg_cin)))
    return terms, bound


def tc_contract(x, w, bias, fmt, dilation=1, pad_left=0, in_act=ACT_NONE, in_slope=0.0, out_act=ACT_NONE, out_slope=0.0, res=None,
                alpha=1.0, y_prev=None, row_lens=None, seg_cin=None):
    """fs2_conv1d on the tensor cores in format fmt ("split3" / "f8"), seg_cin = 256 for the K-segmented tiles.  Returns fp64
    (y_c, y64, S, R): the rounded-operand contract, the unrounded contract, and the scales of the two bars (see above)."""
    terms, bound = _pairs(x, w, fmt, in_act, in_slope, seg_cin)
    lin = lambda pairs: sum(conv1d(a_, w_, None, dilation, pad_left) for a_, w_ in pairs)
    d = lambda t: None if t is None else t.double()
    ab = lambda t: None if t is None else t.double().abs()
    epi = lambda acc: conv1d_epilogue(acc, d(bias), out_act, out_slope, d(res), alpha, d(y_prev), row_lens)
    a64 = act_operand(x, in_act, in_slope).double()
    y64 = conv1d_epilogue(conv1d(a64, w.double(), None, dilation, pad_left), d(bias), out_act, out_slope, d(res), alpha, d(y_prev), row_lens)
    mass = accumulator_mass(terms, dilation, pad_left, seg_cin)
    S = conv1d_epilogue(lin([(a_.abs(), w_.abs()) for a_, w_ in terms]) + mass, ab(bias), ACT_NONE, 0.0, ab(res), abs(alpha), ab(y_prev),
                        row_lens)
    R = conv1d_epilogue(lin(bound), None, ACT_NONE, 0.0, None, abs(alpha), None, row_lens)
    return epi(lin(terms)), y64, S, R


def tc_bound(x, w, fmt, dilation=1, pad_left=0, in_act=ACT_NONE, in_slope=0.0):
    """R of tc_contract before the epilogue (alpha 1), without the other sums."""
    _, bound = _pairs(x, w, fmt, in_act, in_slope, None)
    return sum(conv1d(a_, w_, None, dilation, pad_left) for a_, w_ in bound)


def accumulator_mass(terms, dilation=1, pad_left=0, seg_cin=None):
    """Sum over the K-steps of |running sum| of the accumulator, per output element, in the order the conv kernel walks them (16-channel
    K-block outer, tap inner; conv_tc_kernel.cuh).  K-segmented (seg_cin): every (tap, seg_cin-channel) slice has a fresh accumulator,
    and each slice's fp32 add into y counts |y so far| once more."""
    a0, w0 = terms[0]
    B, T, cin = a0.shape
    taps, _, N = w0.shape
    mass = torch.zeros(B, T, N, dtype=torch.float64)
    y = torch.zeros_like(mass)
    step = lambda tap, c: sum(conv1d(a_[..., c:c + 16], w_[tap:tap + 1, c:c + 16], None, dilation, pad_left - tap * dilation)
                              for a_, w_ in terms)
    slices = [(range(taps), 0, cin)] if seg_cin is None else [([t], c, c + seg_cin) for t in range(taps) for c in range(0, cin, seg_cin)]
    for tap_list, c0, c1 in slices:
        acc = torch.zeros_like(mass)
        for c in range(c0, c1, 16):
            for tap in tap_list:
                acc += step(tap, c)
                mass += acc.abs()
        if seg_cin is not None:
            y += acc
            mass += y.abs()
    return mass


def tc_errors(got, y_c, y64, S, R):
    """The two normalised errors, max over elements: (a) |y - y_c| / (2^-24 S) and (b) max(0, |y - y64| - R) / (2^-24 S).  Where S = 0
    (masked rows, all-zero products) the output must be exact.  Each must stay <= TC_ACC_C."""
    def norm(d):
        r = torch.where(S > 0, d / (U24 * S.clamp_min(1e-300)), torch.where(d > 0, float("inf"), 0.0))
        return torch.nan_to_num(r, nan=float("inf")).max().item()
    g = got.double()
    return norm((g - y_c).abs()), norm(((g - y64).abs() - R).clamp_min(0.0))


def unpack_conv_tc(buf, taps, cin, n, nb):
    """Inverse of packing.pack_conv_tc for a [taps][Cin][N] weight tiled with NB output channels per work item: decodes the header
    (1/s, format) and both planes, and returns the weight side of each term as w_planes does, from the bytes alone."""
    buf = buf.cpu()
    inv_s = float(buf[:4].view(torch.float32))
    fmt = int(buf[4])
    kb, nblk = cin // 16, n // nb
    tiles = buf[128:].reshape(nblk, kb, taps, 2, 2 * nb * 16)

    def f16_plane(p):       # [nblk][kb][tap][chunk][nn][8 halfs] -> [tap][kb * 16 + chunk * 8 + i][nblk * NB + nn]
        h = tiles[:, :, :, p].contiguous().view(torch.float16).reshape(nblk, kb, taps, 2, nb, 8)
        return h.permute(2, 1, 3, 5, 0, 4).reshape(taps, cin, n).double()

    hi = f16_plane(0)
    if fmt == 0:
        return [hi * inv_s, hi * inv_s, f16_plane(1) * inv_s]
    e = tiles[:, :, :, 1].contiguous().reshape(nblk, kb, taps, 2, nb, 16).view(torch.float8_e4m3fn).double()   # [.][h8 | l8][nn][16 ch]
    e4 = lambda c: e[:, :, :, c].permute(2, 1, 4, 0, 3).reshape(taps, cin, n)
    return [hi * inv_s, e4(0) * 4096.0 * inv_s, e4(1) * inv_s]


def resblock_group(x, kernels, dils, w1, b1, w2, b2, conv=conv1d):
    """fs2_resstack as the per-layer calls of model.cu's unfused vocoder path:  r <- conv2(conv1(r, lrelu in / out) ) + r  per
    dilation, the last conv of each kernel size scaled by 1/n_kernels and accumulated into the sum.  w1 / w2 [j][d]: [k][C][C]."""
    nk = len(kernels)
    xs = None
    for j, k in enumerate(kernels):
        r = x
        for d, dv in enumerate(dils[j]):
            t = conv(r, w1[j][d], b1[j][d], dv, (k - 1) * dv // 2, ACT_LRELU, 0.1, ACT_LRELU, 0.1)
            last = d == len(dils[j]) - 1
            r = conv(t, w2[j][d], b2[j][d], 1, (k - 1) // 2, res=r, alpha=1.0 / nk if last else 1.0,
                     y_prev=xs if last and j > 0 else None)
        xs = r
    return xs


def resstack_contract(x, kernels, dils, w1, b1, w2, b2, alpha=None, y_prev=None):
    """fs2_resstack (f16 + f8 operands, intermediates re-split on chip) in fp64 with the two bar scales of the group: S and R summed over
    its layers, each layer's own (S of a conv = conv(|a|, |w|) + |b| on its exact input, R its format bound), plus |x| for the residual.
    Carrying them through the later convs' |w| instead would multiply them by sum |w| (about 9 for the shipped layers) per conv, and
    leave a bar that nothing could fail.  So S and R here are scales, not derived bounds: an early layer's error reaches the output
    through the later convs with a gain this sum ignores.  Bars built on them are empirical (measured constants), and a failure is
    not by itself proof of a kernel bug.  alpha = None: the mean over kernel sizes (the group); else y_prev + alpha * the one kernel
    size.  Returns (y64, S, R) for tc_errors."""
    def layer(v, w, b, dil, pad):
        a = _act(v, ACT_LRELU, 0.1)
        s = conv1d(a.abs(), w.double().abs(), b.double().abs(), dil, pad)
        return conv1d(a, w.double(), b.double(), dil, pad), s, tc_bound(v, w, "f8", dil, pad, ACT_LRELU, 0.1)
    y = S = R = 0.0
    for j, k in enumerate(kernels):
        r, rS, rR = x.double(), x.double().abs(), 0.0
        for d, dv in enumerate(dils[j]):
            t, tS, tR = layer(r, w1[j][d], b1[j][d], dv, (k - 1) * dv // 2)
            u, uS, uR = layer(t, w2[j][d], b2[j][d], 1, (k - 1) // 2)
            r, rS, rR = u + r, rS + tS + uS, rR + tR + uR
        y, S, R = y + r, S + rS, R + rR
    a = 1.0 / len(kernels) if alpha is None else alpha
    y, S, R = a * y, abs(a) * S, abs(a) * R
    if y_prev is not None:
        y, S = y + y_prev.double(), S + y_prev.double().abs()
    return y, S, R


def layernorm(x, g, b, row_lens=None):
    y = torch.nn.functional.layer_norm(x, (x.shape[-1],), g, b, 1e-5)
    if row_lens is not None:
        y = y.masked_fill((torch.arange(x.shape[1])[None, :] >= row_lens[:, None])[..., None], 0.0)
    return y


def attention(qkv, H, key_lens):
    B, T, D3 = qkv.shape
    D = D3 // 3
    dh = D // H
    q, k, v = (qkv[..., i * D:(i + 1) * D].reshape(B, T, H, dh).permute(0, 2, 1, 3) for i in range(3))
    s = (q @ k.transpose(-1, -2)) * (1.0 / math.sqrt(dh))
    s = s.masked_fill((torch.arange(T)[None, :] >= key_lens[:, None])[:, None, None, :], float("-inf"))
    ctx = (torch.softmax(s, -1) @ v).permute(0, 2, 1, 3).reshape(B, T, D)
    return ctx.masked_fill((torch.arange(T)[None, :] >= key_lens[:, None])[..., None], 0.0)


# ------------------------------------------------------------------ the fused attention kernel's operand formats and their bound
#
# attention_fused.cu multiplies fp16 hi / lo operands three MMAs at a time, as the convolutions do (Dh = 128, scale = 128^-1/2):
#   S = Q_lo K_hi + Q_hi K_hi + Q_hi K_lo        Q split as it is, K split x AF_WSCALE = 16 (the packed tiles)
#   p = exp2(S c - m) in fp32, l = the sum of the fp32 p, P = p x AF_PSCALE split into fp16 hi / lo
#   O = (P_lo V_hi + P_hi V_hi + P_hi V_lo) / (16 AF_PSCALE l)        V split x 16
# All converts saturate at +-65504, so the domain is |q| < 65504 and |k|, |v| < 4094; beyond it the operands clip without an error.
#
# R (attention_contract), per output element, bounds |O(rounded Q, K, V) - O64| from the stated precision of the three splits
# (_split3_err: 2^-22 relative, the absolute floor 2^-25 of a subnormal lo; for K and V that floor is 2^-29 after the / 16):
#   score:  q.k - S = q_lo k_lo + q ek + eq k - eq ek with |eq| <= e_q, |ek| <= e_k, so one key's scaled score is off by at most
#           d_s = scale sum_d (|q_lo| |k_lo| + |q| e_k + e_q |k| + e_q e_k).
#   softmax: scores off by eps_s (|eps_s| <= d_s) move O by sum_s w_s (e^eps_s - 1)(v_s - O) / sum_s w_s e^eps_s, w the exact weights:
#           at most e^dmax sum_s w_s expm1(d_s) |v_s - O|.
#   values: the perturbed weights (each <= w_s e^(2 dmax)) times the V error: at most e^(2 dmax) sum_s w_s e_v,s.
# P is not in R.  It lies in (0, 1], and AF_PSCALE = 2^15 keeps its lo plane normal down to p ~ 2^-18, so P costs 2^-22 relative
# (the dropped P_lo V_lo term as much again), which the bar of the tests absorbs.  Without the scale its lo plane is subnormal below
# p ~ 2^-3 and each weight carries up to 2^-25 absolute: on a row whose keys share one score and one value those errors add up n
# times while l, summed from the unrounded p, does not see them.  Charging that floor to R would make the bar vacuous at decoder
# lengths; the kernel must not have it (tests/test_attention_precision_cpu.py).

ATT_PSCALE = 2.0 ** 15       # AF_PSCALE of attention_fused.cu
ATT_WSCALE = 16.0            # AF_WSCALE


def _heads(qkv, H, b, n):
    """q, k, v of utterance b's first n rows, [H][n][dh] each, as qkv's dtype."""
    D = qkv.shape[2] // 3
    return [qkv[b, :n, i * D:(i + 1) * D].reshape(n, H, D // H).transpose(0, 1) for i in range(3)]


def _key_rows(key_lens, T, b):
    return min(max(int(key_lens[b]), 0), T)


def attention_contract(qkv, H, key_lens):
    """The fused kernel's contract in fp64: (o64, R), both [B, T, D], o64 the exact attention (E.attention), R the bound above; both
    zero on padded query rows."""
    B, T, D3 = qkv.shape
    D = D3 // 3
    dh = D // H
    scale = 1.0 / math.sqrt(dh)
    o64 = torch.zeros(B, T, D, dtype=torch.float64)
    R = torch.zeros_like(o64)
    for b in range(B):
        n = _key_rows(key_lens, T, b)
        if n == 0:
            continue
        q, k, v = (t.float() for t in _heads(qkv, H, b, n))
        q64, k64, v64 = q.double(), k.double(), v.double()
        w = torch.softmax(q64 @ k64.transpose(-1, -2) * scale, -1)
        o = w @ v64
        ks, vs = k * ATT_WSCALE, v * ATT_WSCALE
        lo = lambda t: _f16(t - _f16(t)).double().abs()
        lq, lk = lo(q), lo(ks) / ATT_WSCALE
        eq, ek, ev = _split3_err(q), _split3_err(ks) / ATT_WSCALE, _split3_err(vs) / ATT_WSCALE
        d = scale * (torch.cat([lq, q64.abs(), eq, eq], -1) @ torch.cat([lk, ek, k64.abs(), ek], -1).transpose(-1, -2))
        dmax = d.amax(-1, keepdim=True)
        we = w * torch.expm1(d)
        soft = torch.empty_like(o)                     # sum_s we_s |v_s - O|, in row chunks of at most 2^24 (row, key, d) terms
        step = max(1, 2 ** 24 // (n * dh))
        for h in range(H):
            for t0 in range(0, n, step):
                diff = (v64[h][None] - o[h, t0:t0 + step, None]).abs()
                soft[h, t0:t0 + step] = (we[h, t0:t0 + step, None] @ diff)[:, 0]
        r = torch.exp(dmax) * soft + torch.exp(2 * dmax) * (w @ ev)
        o64[b, :n] = o.transpose(0, 1).reshape(n, D)
        R[b, :n] = r.transpose(0, 1).reshape(n, D)
    return o64, R


def attention_fused_emul(qkv, H, key_lens, p_scale=ATT_PSCALE):
    """The fused kernel's arithmetic with exact sums: fp16 splits as split_f16x2 rounds them, S rounded to fp32, p = exp2(S c - m)
    in fp32 as the kernel forms it, l the fp64 sum of those p, P split x p_scale, O summed in fp64.  p_scale = 1 is the kernel
    without AF_PSCALE.  Returns [B, T, D] fp64, zero on padded query rows."""
    B, T, D3 = qkv.shape
    D = D3 // 3
    dh = D // H
    f32 = lambda t: t.float().double()
    c = f32(torch.tensor(dh ** -0.5, dtype=torch.float32) * (1.0 / ATT_WSCALE) * 1.4426950408889634)
    out = torch.zeros(B, T, D, dtype=torch.float64)
    for b in range(B):
        n = _key_rows(key_lens, T, b)
        if n == 0:
            continue
        q, k, v = (t.float() for t in _heads(qkv, H, b, n))
        split = lambda t: (_f16(t), _f16(t - _f16(t)))
        (qh, ql), (kh, kl), (vh, vl) = split(q), split(k * ATT_WSCALE), split(v * ATT_WSCALE)
        mm = lambda a, bt: a.double() @ bt.double()
        s = f32(mm(ql, kh.transpose(-1, -2)) + mm(qh, kh.transpose(-1, -2)) + mm(qh, kl.transpose(-1, -2)))
        sc = f32(s * c)
        m = sc.amax(-1, keepdim=True)
        p = f32(torch.exp2(f32(s * c - m)))
        l = p.sum(-1, keepdim=True)
        ph, pl = split((p * p_scale).float())
        o = (mm(pl, vh) + mm(ph, vh) + mm(ph, vl)) / (ATT_WSCALE * p_scale * l)
        out[b, :n] = o.transpose(0, 1).reshape(n, D)
    return out


def fft_block(pk, pfx, x, lens, H, k1, k2):
    qkv = conv1d(x, pk[pfx + "w_qkv"][None], pk[pfx + "b_qkv"])
    ctx = attention(qkv, H, lens)
    tmp = conv1d(ctx, pk[pfx + "w_o"][None], pk[pfx + "b_o"], res=x)
    x = layernorm(tmp, pk[pfx + "ln1_g"], pk[pfx + "ln1_b"], lens)
    hid = conv1d(x, pk[pfx + "w_1"], pk[pfx + "b_1"], pad_left=(k1 - 1) // 2, out_act=ACT_RELU)
    tmp = conv1d(hid, pk[pfx + "w_2"], pk[pfx + "b_2"], pad_left=(k2 - 1) // 2, res=x)
    return layernorm(tmp, pk[pfx + "ln2_g"], pk[pfx + "ln2_b"], lens)


def variance_head(h, w, b, lens, control, target, bins, emb, x):
    pred = h @ w + b
    pred = pred.masked_fill(torch.arange(h.shape[1])[None, :] >= lens[:, None], 0.0)
    if bins is None:
        return pred, x
    if target is not None:
        key = target
    else:
        pred = pred * control
        key = pred
    idx = (~(bins[None, None, :] >= key[..., None])).sum(-1)    # torch.bucketize(right=False): NaN -> len(bins), like ATen's search
    return pred, x + emb[idx]


def predictor(pk, nm, x, lens, k, control=1.0, target=None, bins=None, emb=None, x_acc=None):
    h = conv1d(x, pk[nm + ".w_c1"], pk[nm + ".b_c1"], pad_left=(k - 1) // 2, out_act=ACT_RELU)
    h = layernorm(h, pk[nm + ".ln1_g"], pk[nm + ".ln1_b"])
    h = conv1d(h, pk[nm + ".w_c2"], pk[nm + ".b_c2"], pad_left=1, out_act=ACT_RELU)
    h = layernorm(h, pk[nm + ".ln2_g"], pk[nm + ".ln2_b"])
    return variance_head(h, pk[nm + ".w_out"], pk[nm + ".b_out"], lens, control, target, bins, emb, x_acc)


def durations(src, use_target, d_control):
    if use_target:
        d = src
        d_rounded = None
    else:
        d = torch.clamp(torch.round(torch.exp(src) - 1) * d_control, min=0)     # torch.clamp keeps NaN
        d_rounded = d
    # the reference's int() raises on NaN and +-inf (a -inf target too); those and durations past 1e6 frames count as wild, 0 frames
    wild = ~((d <= 1.0e6) & (d > -math.inf))
    reps = torch.where(wild, torch.zeros_like(d), d).trunc().clamp(min=0).to(torch.int32)
    cum = torch.cumsum(reps, dim=1).to(torch.int32)
    return d_rounded, cum, cum[:, -1].long(), int(wild.sum())


def length_regulate(x, cum, pos, T):
    B, L, D = x.shape
    t = torch.arange(T, dtype=torch.int32)
    idx = torch.searchsorted(cum, t[None, :].expand(B, T).contiguous(), right=True).clamp(max=L - 1)   # first i with cum[i] > t
    y = torch.gather(x, 1, idx[..., None].expand(B, T, D).long())
    y = y.masked_fill((t[None, :] >= cum[:, -1:])[..., None], 0.0)
    return y + pos[:T]


def acoustic_forward(pk, cfg, speakers, texts, src_lens, p_control=1.0, d_control=1.0, p_target=None, e_target=None,
                     d_target=None, mel_lens=None, max_mel_len=None, pitch_frame=False, energy_frame=False):
    """Mirror of encode_impl + decode_impl in model.cu.  cfg: dict(n_head,k1,k2,n_enc,n_dec,vp_kernel,n_postnet,post_k)."""
    B, L = texts.shape
    lens = src_lens.to(torch.int32)
    x = pk["word_emb"][texts] + pk["enc_pos"][:L]
    for i in range(cfg["n_enc"]):
        x = fft_block(pk, f"enc.{i}.", x, lens, cfg["n_head"], cfg["k1"], cfg["k2"])
    if "spk_emb" in pk:
        x = x + pk["spk_emb"][speakers][:, None, :]
    k = cfg["vp_kernel"]
    logd, _ = predictor(pk, "dur", x, lens, k)
    p_pred = e_pred = None
    if not pitch_frame:
        p_pred, x = predictor(pk, "pitch", x, lens, k, p_control, p_target, pk["pitch_bins"], pk["pitch_emb"], x)
    if not energy_frame:
        e_pred, x = predictor(pk, "energy", x, lens, k, p_control, e_target, pk["energy_bins"], pk["energy_emb"], x)
    d_rounded, cum, mel_len, _ = durations(d_target if d_target is not None else logd, d_target is not None, d_control)
    T = int(max_mel_len) if max_mel_len is not None else int(mel_len.max())
    mask_lens = (mel_lens if mel_lens is not None else mel_len).to(torch.int32)
    if pitch_frame or energy_frame:                  # decode_impl: LR without positions, frame-level heads, then fs2_add_positions
        y = length_regulate(x, cum, torch.zeros_like(pk["dec_pos"]), T)
        if pitch_frame:
            p_pred, y = predictor(pk, "pitch", y, mask_lens, k, p_control, p_target, pk["pitch_bins"], pk["pitch_emb"], y)
        if energy_frame:
            e_pred, y = predictor(pk, "energy", y, mask_lens, k, p_control, e_target, pk["energy_bins"], pk["energy_emb"], y)
        y = y + pk["dec_pos"][:T]
    else:
        y = length_regulate(x, cum, pk["dec_pos"], T)
    for i in range(cfg["n_dec"]):
        y = fft_block(pk, f"dec.{i}.", y, mask_lens, cfg["n_head"], cfg["k1"], cfg["k2"])
    mel = conv1d(y, pk["w_mel"][None], pk["b_mel"])
    cur = mel
    n = cfg["n_postnet"]
    for i in range(n):
        last = i == n - 1
        cur = conv1d(cur, pk[f"post.{i}.w"], pk[f"post.{i}.b"], pad_left=(cfg["post_k"] - 1) // 2,
                     out_act=ACT_NONE if last else ACT_TANH, res=mel if last else None)
    return mel, cur, p_pred, e_pred, logd, d_rounded, mel_len


def vocoder_forward(pk, rates, rb_k, rb_dil, mel_cl):
    """Mirror of fs2_vocoder_forward (model.cu's window_walk over [0, T)).  mel_cl: [B,T,80] channels-last."""
    x = conv1d(mel_cl, pk["w_pre"], pk["b_pre"], pad_left=3)
    nk = len(rb_k)
    for i, u in enumerate(rates):
        B, Ti, C = x.shape
        Co = C // 2
        half = u // 2
        ya = conv1d(x, pk[f"up.{i}.wa"], pk[f"up.{i}.b"][: half * Co], pad_left=1, in_act=ACT_LRELU, in_slope=0.1)
        yb = conv1d(x, pk[f"up.{i}.wb"], pk[f"up.{i}.b"][half * Co:], pad_left=0, in_act=ACT_LRELU, in_slope=0.1)
        xu = torch.cat([ya, yb], dim=-1).reshape(B, Ti * u, Co)       # [B][T][u*Co] viewed as [B][T*u][Co]
        xs = None
        for j in range(nk):
            rb, k = i * nk + j, rb_k[j]
            r = xu
            for d, dil in enumerate(rb_dil[j]):
                t = conv1d(r, pk[f"rb.{rb}.{d}.w1"], pk[f"rb.{rb}.{d}.b1"], dilation=dil, pad_left=(k * dil - dil) // 2,
                           in_act=ACT_LRELU, in_slope=0.1, out_act=ACT_LRELU, out_slope=0.1)
                last = d == len(rb_dil[j]) - 1
                r = conv1d(t, pk[f"rb.{rb}.{d}.w2"], pk[f"rb.{rb}.{d}.b2"], pad_left=(k - 1) // 2, res=r,
                           alpha=(1.0 / nk) if last else 1.0, y_prev=xs if (last and j > 0) else None)
            xs = r
        x = xs
    xa = torch.where(x > 0, x, x * 0.01)
    B, T, C = x.shape
    acc = torch.zeros(B, T)
    for j in range(7):
        shift = j - 3
        lo, hi = max(0, -shift), min(T, T - shift)
        acc[:, lo:hi] += xa[:, lo + shift:hi + shift] @ pk["w_post"][j]
    return torch.tanh(acc + pk["b_post"])
