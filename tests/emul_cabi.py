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
    idx = (bins[None, None, :] < key[..., None]).sum(-1)
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
        d = torch.clamp(torch.round(torch.exp(src) - 1) * d_control, min=0)
        d_rounded = d
    reps = d.trunc().clamp(min=0).to(torch.int32)
    cum = torch.cumsum(reps, dim=1).to(torch.int32)
    return d_rounded, cum, cum[:, -1].long()


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
    d_rounded, cum, mel_len = durations(d_target if d_target is not None else logd, d_target is not None, d_control)
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
    """Mirror of vocoder_impl in model.cu.  mel_cl: [B,T,80] channels-last."""
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
