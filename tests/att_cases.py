"""Attention cases and bars (TEST INFRASTRUCTURE, shared by tests/test_gpu_ops.py, tests/test_gpu_attention_precision.py
and tests/test_attention_precision_cpu.py).

N(0, 1) queries, keys and values give every key its own score and value, so the rounding errors of the fused kernel's operand
splits (tests/emul_cabi.py, above attention_contract) come out with random signs and average away.  The magnitude cases here
make them add up instead: many keys sharing one score and one value (plateau, uniform), values, keys and queries across the
magnitudes the splits represent (vscale, kqscale), and the adversarial score patterns of attention_qkv at scaled operands.
"""
import torch

U24 = 2.0 ** -24
DH = 128
H = 2


def _g(seed):
    return torch.Generator().manual_seed(seed)


def attention_qkv(kind, lens, T, seed=3):
    """qkv [B, T, 768] (2 heads of 128).  "random": N(0, 1).  The others are adversarial for a softmax kernel: every query is
    8 u + small noise for one unit vector u, so a key c u scores about 8 c / sqrt(128) nats against all of them, per utterance of n keys:
      last_tile_max: key n - 1 scores 42 nats, every earlier one |s| < ~3: breaks a missing online-softmax rescale.
      masked_max:    the keys at and past n score 140 nats: breaks a max taken before masking.
      range80:       keys spread over [-80, 50] nats and key n // 2 at +80: the far keys' weights underflow to 0, O = that key's v.
      tied:          keys 0 and n - 1 (different 64-key tiles) share the row max bit for bit: O = the mean of their v."""
    B = len(lens)
    if kind == "random":
        return torch.randn(B, T, 768, generator=_g(seed))
    gen = _g(seed)
    u = torch.ones(DH) / DH ** 0.5
    q = 8 * u + 0.01 * torch.randn(B, T, 2, DH, generator=gen)
    k = torch.randn(B, T, 2, DH, generator=gen)
    v = torch.randn(B, T, 2, DH, generator=gen)
    nats = lambda s: s * DH ** 0.5 / 8 * u
    for b, n in enumerate(lens):
        n = min(max(n, 0), T)
        if n == 0:
            continue
        if kind == "last_tile_max":
            k[b, n - 1] = nats(42.0)
        elif kind == "masked_max":
            k[b, n:] = nats(140.0)
        elif kind == "range80":
            s = torch.rand(T, 2, 1, generator=gen, dtype=torch.float64).float() * 130 - 80
            k[b] = s * nats(1.0)
            k[b, n // 2] = nats(80.0)
        elif kind == "tied":
            k[b] = 0.1 * k[b]
            k[b, 0] = nats(30.0)
            k[b, n - 1] = nats(30.0)
    return torch.cat([q.reshape(B, T, 256), k.reshape(B, T, 256), v.reshape(B, T, 256)], dim=2)


def attention_bar_scale(qkv, key_lens):
    """Per (utterance, query row, head): max_s |v_s| (1 + scale max_s sum_d |q_d| |k_sd|) over the valid keys s, in fp64."""
    B, T, _ = qkv.shape
    q, k, v = (qkv[..., i * 256:(i + 1) * 256].double().abs().reshape(B, T, 2, 128).permute(0, 2, 1, 3) for i in range(3))
    valid = (torch.arange(T)[None, :] < key_lens.clamp(0, T)[:, None])[:, None, :, None]     # [B, 1, Tk, 1]
    vmax = (v * valid).amax(dim=(2, 3))                                                    # [B, H]
    qk = (q @ k.transpose(-1, -2)).masked_fill(~valid.transpose(-1, -2), 0.0).amax(dim=-1)   # [B, H, T]
    return (vmax[..., None] * (1 + qk / 128 ** 0.5)).permute(0, 2, 1)                    # [B, T, H]


def attention_normalised_err(got, want, scale, R=None):
    """max over rows of max_d max(0, |got - want| - R) / (2^-24 scale_row); rows of zero scale (no valid key) must be exact."""
    B, T, _ = got.shape
    d = (got.double() - want).abs()
    if R is not None:
        d = (d - R).clamp_min(0.0)
    d = d.reshape(B, T, 2, 128).amax(-1)
    r = torch.where(scale > 0, d / (U24 * scale.clamp_min(1e-300)), torch.where(d > 0, float("inf"), 0.0))
    return torch.nan_to_num(r, nan=float("inf")).max().item()


# per-row error bar of both attention backends in units of 2^-24 max|v| (1 + scale max sum|q||k|) (attention_bar_scale), after R
# for the fused kernel (tests/emul_cabi.py::attention_contract; the exact kernel's operands are fp32, R = 0).  Largest values measured
# on an H100 80GB HBM3 (700 W power limit), re-measured with the exact kernel's compensated sums: over test_gpu_ops' ATT_ADV_CASES and
# ATT_DECODER_CASES 0.53 for the exact kernel (0.41 before, on fewer cases) and 3.9 for the fused one (the range80 rows, O against
# the argmax key's v; 1.07 over the others); over CASES below, plateau aside, 0.68 for the exact kernel (V in [2048, 4094)) and 4.97
# for the fused one after R (pfloor at 4200 keys).  The plateau rows are known failures (test_gpu_attention_precision).
ATT_EXACT_C = {0: 2.0, 2: 16.0}

# ------------------------------------------------------------------ magnitude cases: (name, family, parameter, T, lens)
# plateau: per utterance of n keys, one dominant key (index n // 3) and n - 1 keys with one K row and one V row (N(0, 1) values, so
#   not fp16 numbers); query row t scores the dominant key gap_t / 2 nats above 0 and the plateau gap_t / 2 below, gap_t from a
#   grid of 32 gaps in [2, 16] nats (shifted by half a step in the second head), so that some p = e^-gap lands near the worst lo
#   rounding.  The bar scale is then max|v| (1 + gap / 2).
# pfloor: the plateau with gaps in [12, 16] nats and a zero V row on the dominant key.  Every plateau weight p < 2^-17 then sits
#   where an unscaled fp16 split of p has a subnormal hi and lo (2^-25 absolute, 2^-8 relative), while the accumulator holds only
#   the plateau's products, so the tensor cores' truncation against it stays far below that floor: the row that tells a kernel
#   without AF_PSCALE from one with it.
# vscale: V = N(0, 1) 2^e, or |v| uniform in [2048, 4094) (the top of the V domain), or N(0, 1) times a per-channel 2^u, u uniform
#   in [-16, 8]; Q, K N(0, 1).
# kqscale: K 2^e and Q 2^-e (the scores do not change), e = -8 .. 8.
# uniform: one K row per utterance, so every score of a row is equal and l = n.
# adv: attention_qkv's range80 / tied / masked_max rows with K and V times 2^e and Q times 2^-e.
EDGE_LENS = [0, 1, 63, 64, 65, 127, 128, 129, 300, 10 ** 6, -3]            # T = 300: plus one past T and one negative (both clamped)


def _lens(T):
    return [T, 129, 128, 127]


PLATEAU_GAPS = 32
CASES = (
    [(f"plateau_T{T}", "plateau", None, T, _lens(T)) for T in (300, 1012, 4200)]
    + [(f"pfloor_T{T}", "pfloor", None, T, _lens(T)) for T in (1012, 4200)]
    + [(f"vscale_2^{e}", "vscale", ("scale", e), 1012, _lens(1012)) for e in (-16, -12, -8, -4, 0, 4, 8)]
    + [("vscale_[2048,4094)", "vscale", ("band", 2048.0, 4094.0), 1012, _lens(1012)),
       ("vscale_chan2^-16..2^8", "vscale", ("chan", -16, 8), 1012, _lens(1012))]
    + [(f"kqscale_2^{e}", "kqscale", e, 300, _lens(300)) for e in range(-8, 9)]
    + [("uniform_T4200", "uniform", None, 4200, [4200, 4097, 129, 127])]
    + [(f"adv_{kind}_2^{e}", "adv", (kind, e), 300, EDGE_LENS) for kind in ("range80", "tied", "masked_max") for e in (-8, 8)]
)
FAMILIES = ("plateau", "pfloor", "vscale", "kqscale", "uniform", "adv")


def _plateau(T, lens, seed, gap0=2.0, gap1=16.0, zero_dom=False):
    B = len(lens)
    scale = DH ** -0.5
    c = 4.0                                            # |k| = c: the dominant key c u, the plateau -c u
    step = (gap1 - gap0) / (PLATEAU_GAPS - 1)
    q = torch.randn(B, T, H, DH, generator=_g(seed))
    k = torch.randn(B, T, H, DH, generator=_g(seed + 1))
    v = torch.randn(B, T, H, DH, generator=_g(seed + 2))
    gen = _g(seed + 3)
    for b, n in enumerate(lens):
        n = min(max(n, 0), T)
        for h in range(H):
            u = torch.randn(DH, generator=gen)
            u = u / u.norm()
            gaps = gap0 + step * (torch.arange(T) % PLATEAU_GAPS + 0.5 * h)
            q[b, :, h] = (gaps / (2 * scale * c))[:, None] * u
            if n == 0:
                continue
            k[b, :n, h] = -c * u
            v[b, :n, h] = torch.randn(DH, generator=gen)
            j = n // 3
            k[b, j, h] = c * u
            v[b, j, h] = 0.0 if zero_dom else torch.randn(DH, generator=gen)
    return torch.cat([t.reshape(B, T, H * DH) for t in (q, k, v)], dim=2)


def _signed_band(shape, lo, hi, seed):
    m = lo + (hi - lo) * torch.rand(*shape, generator=_g(seed), dtype=torch.float64)
    s = torch.where(torch.rand(*shape, generator=_g(seed + 1)) < 0.5, -1.0, 1.0)
    return (m * s).float()


def make_qkv(case, seed=5):
    """qkv [B, T, 768] fp32 of a CASES entry."""
    _, fam, par, T, lens = case
    B = len(lens)
    if fam == "plateau":
        return _plateau(T, lens, seed)
    if fam == "pfloor":
        return _plateau(T, lens, seed, 12.0, 16.0, zero_dom=True)
    if fam == "adv":
        kind, e = par
        qkv = attention_qkv(kind, lens, T)
        return torch.cat([qkv[..., :256] * 2.0 ** -e, qkv[..., 256:] * 2.0 ** e], dim=2)
    q, k, v = (torch.randn(B, T, H * DH, generator=_g(seed + i)) for i in range(3))
    if fam == "vscale":
        if par[0] == "scale":
            v = v * 2.0 ** par[1]
        elif par[0] == "band":
            v = _signed_band((B, T, H * DH), par[1], par[2], seed + 7)
        else:
            v = v * torch.exp2(par[1] + (par[2] - par[1]) * torch.rand(H * DH, generator=_g(seed + 9)))
    elif fam == "kqscale":
        q, k = q * 2.0 ** -par, k * 2.0 ** par
    elif fam == "uniform":
        k = k[:, :1].expand(B, T, H * DH).contiguous()
    else:
        raise ValueError(case)
    return torch.cat([q, k, v], dim=2)


def key_lens(case):
    return torch.tensor(case[4], dtype=torch.int32)


def scores(qkv, kl, got, o64, R):
    """(normalised error after R, max R in the bar's units) of got against the contract, over every row."""
    scale = attention_bar_scale(qkv, kl)
    B, T, _ = got.shape
    r = (R.reshape(B, T, 2, 128).amax(-1) / (U24 * scale.clamp_min(1e-300))).masked_fill(scale == 0, 0.0)
    return attention_normalised_err(got, o64, scale, R), r.max().item()
