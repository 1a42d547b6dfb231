"""Weight re-layout for the sm_90a kernels (pure tensor permutations, device-agnostic, run once per load).

Inputs are reference-keyed tensors (SURVEY.md Appendix C); outputs are the layouts include/fs2b200.h documents:
conv / linear weights as [taps][C_in][C_out] (C_out contiguous), QKV concatenated, eval BatchNorm folded into the
PostNet convs, weight-norm folded, ConvTranspose1d split into its two 2-tap phase groups.
"""
from __future__ import annotations

import math
from typing import Callable, Dict

import torch

Tensor = torch.Tensor


def conv_w(w: Tensor) -> Tensor:
    """nn.Conv1d weight [C_out, C_in, k] -> [k][C_in][C_out]."""
    return w.permute(2, 1, 0).contiguous()


def lin_w(w: Tensor) -> Tensor:
    """nn.Linear weight [out, in] -> [in][out]."""
    return w.t().contiguous()


def conv_tc_block(n_out: int, nb_max: int = 128) -> int:
    """Output channels per work item of the tensor-core kernel (mirror of conv_tc_nb in csrc/conv_tc.cu); 0 = unsupported.
    The f8 split uses nb_max = 64 (its correction term needs an accumulator of its own)."""
    if n_out % 16:
        return 0
    if n_out <= nb_max:
        return n_out
    for nb in range(nb_max, 15, -16):
        if n_out % nb == 0:
            return nb
    return 0


TC_HEADER_BYTES = 128


def split_fp16(w: Tensor):
    """Per-layer power-of-two scale s and the split s*w = hi + lo, hi = fp16(s*w), lo = fp16(s*w - hi)  (s*w - hi is exact
    in fp32).  s puts max|s*w| in [8192, 16384] so that lo stays in fp16's normal range; 1/s is applied in the epilogue."""
    m = float(w.abs().max())
    s = 1.0 if m == 0.0 or not math.isfinite(m) else 2.0 ** math.floor(math.log2(16384.0 / m))
    ws = w.float() * s
    hi = ws.half()
    lo = (ws - hi.float()).half()
    return hi, lo, s


F8_W_HI_SCALE = 2.0 ** -12      # weight hi -> E4M3 (pairs with the kernel's activation-lo scale 2^12, conv_tc_kernel.cuh)
F8_W_LO_SCALE = 1.0             # weight lo -> E4M3 (pairs with the unscaled activation hi)


def _e4m3_bytes(x: Tensor) -> Tensor:
    """fp32 -> E4M3 (round to nearest, saturating at +-448) as uint8."""
    return x.float().clamp(-448.0, 448.0).to(torch.float8_e4m3fn).view(torch.uint8)


def pack_conv_tc(w: Tensor, f8: bool = False, nb: int | None = None):
    """[taps][Cin][N] fp32 -> byte buffer for the tensor-core kernel (see include/fs2b200.h):
         128-byte header (float32[0] = 1/scale, int32[1] = format)  |  [N/NB][Cin/16][taps][2 planes][2 K-chunks][NB][16 bytes]
    Every (tap, 16-channel K-block) stage is one contiguous 64*NB-byte smem image (no-swizzle K-major).
      f8 = False (format 0): plane 0 = fp16 hi, plane 1 = fp16 lo; a chunk row holds 8 channels.
      f8 = True  (format 1, FS2_TC_VARIANT_F8): plane 0 = fp16 hi; plane 1 = E4M3 with chunk 0 = hi * 2^-12 and chunk 1 = lo of the
        K-block's 16 channels -- the B operand of one K = 32 E4M3 MMA against the activations' [lo * 2^12 | hi]; NB <= 64.
    Returns None when the shape is not served by the tensor-core kernel."""
    taps, cin, n = w.shape
    if nb is None:
        nb = conv_tc_block(n, 64 if f8 else 128)
    elif n % nb or nb % 16:
        return None
    if nb == 0 or cin % 16:
        return None
    hi, lo, s = split_fp16(w)
    kb, nblk = cin // 16, n // nb
    hi_t = hi.reshape(taps, kb, 2, 8, nblk, nb).permute(4, 1, 0, 2, 5, 3).contiguous()          # [nblk][kb][tap][chunk][nn][8 halfs]
    plane0 = hi_t.view(torch.uint8).reshape(nblk, kb, taps, 1, 2 * nb * 16)
    if f8:
        ws = w.float() * s
        lo32 = ws - hi.float()                                                                   # exact remainder (not re-rounded to fp16)
        h8 = _e4m3_bytes(hi.float() * F8_W_HI_SCALE).reshape(taps, kb, 16, nblk, nb).permute(3, 1, 0, 4, 2)   # [nblk][kb][tap][nn][16]
        l8 = _e4m3_bytes(lo32 * F8_W_LO_SCALE).reshape(taps, kb, 16, nblk, nb).permute(3, 1, 0, 4, 2)
        plane1 = torch.stack([h8, l8], dim=3).contiguous().reshape(nblk, kb, taps, 1, 2 * nb * 16)
    else:
        lo_t = lo.reshape(taps, kb, 2, 8, nblk, nb).permute(4, 1, 0, 2, 5, 3).contiguous()
        plane1 = lo_t.view(torch.uint8).reshape(nblk, kb, taps, 1, 2 * nb * 16)
    tiles = torch.cat([plane0, plane1], dim=3).contiguous()
    header = torch.zeros(TC_HEADER_BYTES // 4, dtype=torch.float32, device=w.device)
    header[0] = 1.0 / s
    hb = header.view(torch.uint8).clone()
    hb[4] = 1 if f8 else 0
    return torch.cat([hb, tiles.reshape(-1)])


SEG_CIN = 256          # input channels per K-segment of the encoder / predictor path (16 K-steps of the tensor core)


def pack_conv_tc_segments(w: Tensor):
    """[taps][Cin][N] -> taps * (Cin / 256) tile buffers back to back, segment (tap, kc) at index tap * (Cin/256) + kc: a one-tap conv
    over 256 input channels each, three-MMA split, 64 output channels per work item (FS2_TC_VARIANT_NB64).  Every segment carries
    its own power-of-two scale header and is 128 + 1024 * N bytes.  None if the shape does not qualify."""
    taps, cin, n = w.shape
    if cin % SEG_CIN or n % 64:
        return None
    segs = []
    for tap in range(taps):
        for kc in range(cin // SEG_CIN):
            t = pack_conv_tc(w[tap:tap + 1, kc * SEG_CIN:(kc + 1) * SEG_CIN, :].contiguous(), nb=64)
            assert t is not None and t.numel() == 128 + 1024 * n
            segs.append(t)
    return torch.cat(segs)


def add_tc_tiles(pk: Dict[str, Tensor], keys, f8_keys=()) -> None:
    """For every packed conv weight key in `keys` add '<key>_tc' when the tensor-core kernel can take it; keys also listed in
    `f8_keys` get the f16 + f8 operand format."""
    f8_keys = set(f8_keys)
    for k in keys:
        w = pk[k]
        if w.dim() == 2:
            w = w[None]
        t = pack_conv_tc(w, f8=k in f8_keys)
        if t is not None:
            pk[k + "_tc"] = t


def pack_fft_block(g: Callable[[str], Tensor], pfx: str) -> Dict[str, Tensor]:
    a, f = pfx + ".slf_attn.", pfx + ".pos_ffn."
    return {
        "w_qkv": torch.cat([lin_w(g(a + "w_qs.weight")), lin_w(g(a + "w_ks.weight")), lin_w(g(a + "w_vs.weight"))], dim=1).contiguous(),
        "b_qkv": torch.cat([g(a + "w_qs.bias"), g(a + "w_ks.bias"), g(a + "w_vs.bias")]).contiguous(),
        "w_o": lin_w(g(a + "fc.weight")), "b_o": g(a + "fc.bias").contiguous(),
        "ln1_g": g(a + "layer_norm.weight").contiguous(), "ln1_b": g(a + "layer_norm.bias").contiguous(),
        "w_1": conv_w(g(f + "w_1.weight")), "b_1": g(f + "w_1.bias").contiguous(),
        "w_2": conv_w(g(f + "w_2.weight")), "b_2": g(f + "w_2.bias").contiguous(),
        "ln2_g": g(f + "layer_norm.weight").contiguous(), "ln2_b": g(f + "layer_norm.bias").contiguous(),
    }


def pack_predictor(g: Callable[[str], Tensor], pfx: str) -> Dict[str, Tensor]:
    c = pfx + ".conv_layer."
    return {
        "w_c1": conv_w(g(c + "conv1d_1.conv.weight")), "b_c1": g(c + "conv1d_1.conv.bias").contiguous(),
        "ln1_g": g(c + "layer_norm_1.weight").contiguous(), "ln1_b": g(c + "layer_norm_1.bias").contiguous(),
        "w_c2": conv_w(g(c + "conv1d_2.conv.weight")), "b_c2": g(c + "conv1d_2.conv.bias").contiguous(),
        "ln2_g": g(c + "layer_norm_2.weight").contiguous(), "ln2_b": g(c + "layer_norm_2.bias").contiguous(),
        "w_out": g(pfx + ".linear_layer.weight")[0].contiguous(), "b_out": g(pfx + ".linear_layer.bias").contiguous(),
    }


def fold_batchnorm(w: Tensor, b: Tensor, gamma: Tensor, beta: Tensor, mean: Tensor, var: Tensor, eps: float = 1e-5):
    """Conv1d followed by eval-mode BatchNorm1d == one conv (transformer/Layers.py:94,110,125).  fp64 fold, rounded once."""
    scale = gamma.double() / torch.sqrt(var.double() + eps)
    wf = (w.double() * scale[:, None, None]).float()
    bf = ((b.double() - mean.double()) * scale + beta.double()).float()
    return wf, bf


def pack_acoustic(g: Callable[[str], Tensor], n_enc: int, n_dec: int, n_postnet: int, multi_speaker: bool,
                  f8_decoder: bool = False, f8_postnet: bool = False, segmented_encoder: bool = True) -> Dict[str, Tensor]:
    pk: Dict[str, Tensor] = {
        "word_emb": g("encoder.src_word_emb.weight").contiguous(),
        "enc_pos": g("encoder.position_enc")[0].contiguous(),
        "dec_pos": g("decoder.position_enc")[0].contiguous(),
        "pitch_bins": g("variance_adaptor.pitch_bins").contiguous(),
        "energy_bins": g("variance_adaptor.energy_bins").contiguous(),
        "pitch_emb": g("variance_adaptor.pitch_embedding.weight").contiguous(),
        "energy_emb": g("variance_adaptor.energy_embedding.weight").contiguous(),
        "w_mel": lin_w(g("mel_linear.weight")), "b_mel": g("mel_linear.bias").contiguous(),
    }
    if multi_speaker:
        pk["spk_emb"] = g("speaker_emb.weight").contiguous()
    for i in range(n_enc):
        for k, v in pack_fft_block(g, f"encoder.layer_stack.{i}").items():
            pk[f"enc.{i}.{k}"] = v
    for i in range(n_dec):
        for k, v in pack_fft_block(g, f"decoder.layer_stack.{i}").items():
            pk[f"dec.{i}.{k}"] = v
    for nm in ("dur", "pitch", "energy"):
        full = {"dur": "duration", "pitch": "pitch", "energy": "energy"}[nm]
        for k, v in pack_predictor(g, f"variance_adaptor.{full}_predictor").items():
            pk[f"{nm}.{k}"] = v
    for i in range(n_postnet):
        p = f"postnet.convolutions.{i}"
        wf, bf = fold_batchnorm(g(p + ".0.conv.weight"), g(p + ".0.conv.bias"), g(p + ".1.weight"), g(p + ".1.bias"),
                                g(p + ".1.running_mean"), g(p + ".1.running_var"))
        pk[f"post.{i}.w"], pk[f"post.{i}.b"] = conv_w(wf), bf.contiguous()
    tc_keys = [f"{side}.{i}.{w}" for side, n in (("enc", n_enc), ("dec", n_dec)) for i in range(n) for w in ("w_qkv", "w_o", "w_1", "w_2")]
    seg_keys = [k for k in tc_keys if k.startswith("enc.")] + [f"{nm}.{w}" for nm in ("dur", "pitch", "energy") for w in ("w_c1", "w_c2")]
    tc_keys = [k for k in tc_keys if not k.startswith("enc.")]
    post_keys = ["w_mel"] + [f"post.{i}.w" for i in range(n_postnet)]
    f8 = ([k for k in tc_keys if k.startswith("dec.")] if f8_decoder else []) + (post_keys if f8_postnet else [])
    add_tc_tiles(pk, tc_keys + post_keys, f8)
    for k in seg_keys:                       # encoder + predictors: K-segmented tiles (fs2_acoustic_model comment in fs2b200.h)
        w = pk[k]
        t = pack_conv_tc_segments(w[None] if w.dim() == 2 else w) if segmented_encoder else None
        if t is not None:
            pk[k + "_tc"] = t
    return pk


def fold_weight_norm(v: Tensor, gain: Tensor) -> Tensor:
    """w = g * v / ||v||, norm over every dim but 0 (torch weight_norm dim=0; dim 0 is C_in for ConvTranspose1d)."""
    nrm = v.reshape(v.shape[0], -1).norm(dim=1).reshape(gain.shape)
    return v * (gain / nrm)


def split_conv_transpose(w: Tensor, u: int):
    """ConvTranspose1d(k = 2u, stride u, padding u/2) weight [C_in, C_out, k] -> two 2-tap phase-group conv weights.

    out[q*u + p] = sum_t x[t] . W[:, :, (q - t)*u + p + u/2].  With r = p + u/2:
      p <  u/2 (r <  u): taps x[q-1] * W[..., r+u] and x[q]   * W[..., r]      -> group A, conv pad_left = 1
      p >= u/2 (r >= u): taps x[q]   * W[..., r]   and x[q+1] * W[..., r-u]    -> group B, conv pad_left = 0
    Output column (p - p0)*C_out + n of group g lands at element p*C_out + n of the [B][T][u*C_out] == [B][T*u][C_out] row."""
    cin, cout, k = w.shape
    if k != 2 * u or u % 2:
        raise ValueError("needs kernel = 2*stride and even stride")
    half = u // 2
    wa = w.new_empty(2, cin, half * cout)
    wb = w.new_empty(2, cin, half * cout)
    for p in range(half):
        r = p + half
        wa[0, :, p * cout:(p + 1) * cout] = w[:, :, r + u]
        wa[1, :, p * cout:(p + 1) * cout] = w[:, :, r]
    for p in range(half, u):
        r = p + half
        wb[0, :, (p - half) * cout:(p - half + 1) * cout] = w[:, :, r]
        wb[1, :, (p - half) * cout:(p - half + 1) * cout] = w[:, :, r - u]
    return wa.contiguous(), wb.contiguous()


def pack_vocoder(w_of: Callable[[str], Tensor], b_of: Callable[[str], Tensor], rates, n_resblocks: int, n_dil: int,
                 f8_mask: int = 0) -> Dict[str, Tensor]:
    """`w_of(base)` returns the folded weight of conv `base`, `b_of(base)` its bias.  f8_mask: bit 0 = conv_pre, bit 1+i = every conv of
    upsample stage i uses the f16 + f8 operand format (fs2_vocoder_model.f8_mask)."""
    pk: Dict[str, Tensor] = {"w_pre": conv_w(w_of("conv_pre")), "b_pre": b_of("conv_pre").contiguous()}
    for i, u in enumerate(rates):
        wa, wb = split_conv_transpose(w_of(f"ups.{i}"), u)
        pk[f"up.{i}.wa"], pk[f"up.{i}.wb"] = wa, wb
        pk[f"up.{i}.b"] = b_of(f"ups.{i}").repeat(u).contiguous()
    for rb in range(n_resblocks):
        for d in range(n_dil):
            pk[f"rb.{rb}.{d}.w1"] = conv_w(w_of(f"resblocks.{rb}.convs1.{d}"))
            pk[f"rb.{rb}.{d}.b1"] = b_of(f"resblocks.{rb}.convs1.{d}").contiguous()
            pk[f"rb.{rb}.{d}.w2"] = conv_w(w_of(f"resblocks.{rb}.convs2.{d}"))
            pk[f"rb.{rb}.{d}.b2"] = b_of(f"resblocks.{rb}.convs2.{d}").contiguous()
    pk["w_post"] = w_of("conv_post")[0].t().contiguous()      # [1, C, 7] -> [7][C]
    pk["b_post"] = b_of("conv_post").contiguous()
    nk = n_resblocks // len(rates)
    keys = ["w_pre"] + [f"up.{i}.{g}" for i in range(len(rates)) for g in ("wa", "wb")] \
        + [f"rb.{rb}.{d}.{w}" for rb in range(n_resblocks) for d in range(n_dil) for w in ("w1", "w2")]

    def stage_of(k):
        if k == "w_pre":
            return -1
        idx = int(k.split(".")[1])
        return idx if k.startswith("up.") else idx // nk
    add_tc_tiles(pk, keys, [k for k in keys if f8_mask & (1 << (stage_of(k) + 1))])
    return pk
