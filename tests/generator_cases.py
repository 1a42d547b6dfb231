"""Eight HiFi-GAN generators per config that differ where the multi-generator pool's kernels look, and the pools that drive the pool
into the plans large pools pick (TEST INFRASTRUCTURE, shared by tests/test_stream_multi_plans_cpu.py and
tests/test_gpu_stream_multi_plans.py).

In the multi-generator pool (Generator.stream_pool(generators=...), fs2_vocoder_forward_streams_multi) every work item reads its
tiles, weight-scale header and bias from its own stream's generator.  A test sees a generator mix-up only where the generators differ,
so these differ in what the kernels read per generator, not only in their random draws:
  * every generator has its own seed, so its tiles, fp32 weights and biases differ from every other's;
  * every tensor-core layer's packed header (packing.pack_conv_tc's 1 / scale, the power of two that puts max|w| in [8192, 16384))
    differs between every pair of generators, and within a generator each ResBlock conv's header differs from those of its neighbouring
    slots (rb +- 1, d +- 1, the pair's other conv).  Synthetic seeds alone give most layers the same header in every generator.
The headers are moved by rescalings that leave each generator's function unchanged in real arithmetic (LeakyReLU is positively
homogeneous): stage i's signal by 2^a_i (conv_pre's weight and bias by 2^a_-1, ups_i's weight by 2^(a_i - a_(i-1)) and its bias by
2^a_i, conv_post's weight by 2^-a_last) and each ResBlock pair's intermediate by 2^e (convs1's weight by 2^e and bias by 2^(a_i + e),
convs2's weight by 2^-e).  Powers of two scale the folded weight-norm weights exactly, so a rescaled generator's fp64 oracle output
equals its seed's to fp64 rounding.  The ranges of a_i, e and a_i + e are A_RANGE, E_RANGE and AE_RANGE below."""
import ctypes
import itertools
import math

import torch

from fastspeech2_b200 import _lib as L, configs, packing, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from tests import conv_group_cases as G
from tests.test_conv_groups_cpu import vocoder_convs

MAX_GENERATORS = L.MAX_GENERATORS
SEEDS = tuple(201 + k for k in range(MAX_GENERATORS))
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
# log2 ranges of the stage scales a_i, the pair scales e and the pairs' intermediates a_i + e.  Upward every activation stays within 2^4
# of its seed's, where the f16 + f8 split's E4M3 planes ([lo * 2^12 | hi], at most 448) still hold it; downward the tensor-core convs are
# validated to 2^-12 (tests/conv_group_cases.py, x2^-12).  conv_pre's header takes a_-1 alone, so a_i spans 9 values; the 8 pair scales of
# one (ResBlock, dilation) must all differ and be non-zero where every seed gives the pair's two convs the same header (V2's later stages).
A_RANGE, E_RANGE, AE_RANGE = (-5, 3), (-6, 4), (-8, 4)
# the pool policies of tests/test_gpu_stream_multi.py, and V2's 16- and 8-channel stages as fused pairs (d0 > 0 at the narrow widths)
POLICIES = {"default": {}, "exact": {"use_tensor_cores": False}, "per_layer": {"fused_mask": 0, "pair_mask": 0},
            "wide_pairs": {"wide_pairs": True}, "pairs": {"fused_mask": 0, "pair_mask": 0b1111}}
CFG_POLICIES = [("v1", p) for p in ("default", "exact", "per_layer", "wide_pairs")] + [("v2", p) for p in ("default", "exact", "per_layer",
                                                                                                          "pairs")]


def gen_of(b):
    """The generator of stream b: every index, in a pattern with no simple relation to b."""
    return (5 * b + 3) % MAX_GENERATORS


# ---------------------------------------------------------------- the generators
def _folded(sd):
    from oracle import fs2_oracle as O
    return O.fold_weight_norm(sd)


def _hd(cfg):
    h = AttrDict(CFGS[cfg])
    return h, len(h.upsample_rates), len(h.resblock_kernel_sizes), len(h.resblock_dilation_sizes[0])


def _policy_generator(cfg, policy):
    """A CPU Generator of cfg with policy's attributes (its masks; no weights are read)."""
    g = Generator(AttrDict(CFGS[cfg]))
    g.eval()
    for k, v in POLICIES[policy].items():
        setattr(g, k, v)
    return g


def pack(sd, cfg, policy="default"):
    """packing.pack_vocoder of a (weight-normed) state dict as Generator._pack packs it under policy."""
    h, n_st, n_k, n_dil = _hd(cfg)
    g = _policy_generator(cfg, policy)
    f8, _, pair, _ = g.effective_masks()
    wide = [f"rb.{i * n_k + j}.{d}.{w}" for i in range(n_st) if (pair >> (8 + i)) & 1 for j in range(n_k)
            if h.resblock_kernel_sizes[j] <= g.pair_kmax for d in range(n_dil) for w in ("w1", "w2")]
    fw = _folded(sd)
    return packing.pack_vocoder(lambda b: fw[b + ".weight"].float(), lambda b: fw[b + ".bias"].float(), h.upsample_rates, n_st * n_k,
                                n_dil, f8_mask=f8, wide_keys=wide if g.use_tensor_cores else ())


def header_exp(t):
    """log2 of a packed tensor-core buffer's weight-scale header (float32 [0] = 1 / scale)."""
    return int(math.log2(float(t[:4].view(torch.float32)[0])))


def _base_exps(fw, cfg):
    """{packed tensor-core key: log2 of its header} of folded weights fw, from the weights alone (packing.split_fp16's scale)."""
    h, n_st, n_k, n_dil = _hd(cfg)
    exp = lambda w: -int(math.log2(packing.split_fp16(w)[2]))
    out = {"w_pre": exp(fw["conv_pre.weight"])}
    for i, u in enumerate(h.upsample_rates):
        wa, wb = packing.split_conv_transpose(fw[f"ups.{i}.weight"], u)
        if wa.shape[2] % 16 == 0:                      # a phase group of N % 16 != 0 output channels has no tiles
            out[f"up.{i}.wa"], out[f"up.{i}.wb"] = exp(wa), exp(wb)
    for rb in range(n_st * n_k):
        for d in range(n_dil):
            out[f"rb.{rb}.{d}.w1"] = exp(fw[f"resblocks.{rb}.convs1.{d}.weight"])
            out[f"rb.{rb}.{d}.w2"] = exp(fw[f"resblocks.{rb}.convs2.{d}.weight"])
    return out


def _neighbours(key, n_k, n_dil):
    """The ResBlock conv slots next to rb.<rb>.<d>.w<c> in a fused launch's table: rb +- 1 of the same stage, d +- 1 and the pair's other
    conv."""
    _, rb, d, w = key.split(".")
    rb, d = int(rb), int(d)
    out = [f"rb.{rb}.{d}.{'w2' if w == 'w1' else 'w1'}"]
    out += [f"rb.{r}.{d}.{w}" for r in (rb - 1, rb + 1) if r // n_k == rb // n_k]
    out += [f"rb.{rb}.{e}.{w}" for e in (d - 1, d + 1) if 0 <= e < n_dil]
    return out


def _exponents(cfg):
    """The rescaling exponents of the 8 generators: [{'a': [a_-1, a_0, ..], 'e': {(rb, d): e}}], found by a search that makes every
    tensor-core header differ between every pair of generators and from its neighbouring slots within a generator."""
    _, n_st, n_k, n_dil = _hd(cfg)
    base = [_base_exps(_folded(sd), cfg) for sd in seed_state_dicts(cfg)]
    hdr = [dict() for _ in SEEDS]                      # the headers assigned so far
    out = [{"a": [], "e": {}} for _ in SEEDS]
    # variables in launch order: (name, {key: sign}); a stage variable moves its layers' headers by a_i - a_(i-1)
    var = [("a", {"w_pre": 1})]
    for i in range(n_st):
        var.append(("a", {k: 1 for k in (f"up.{i}.wa", f"up.{i}.wb") if k in base[0]}))
        var += [(("e", rb, d), {f"rb.{rb}.{d}.w1": 1, f"rb.{rb}.{d}.w2": -1}) for rb in range(i * n_k, (i + 1) * n_k) for d in range(n_dil)]

    def ok(k, keys, x):
        new = {key: base[k][key] + sign * x for key, sign in keys.items()}
        for key, v in new.items():
            if any(hdr[q].get(key) == v for q in range(len(SEEDS)) if q != k):
                return False
            if key.startswith("rb.") and any(dict(hdr[k], **new).get(n) == v for n in _neighbours(key, n_k, n_dil)):
                return False
        return True

    def domain(k, name):
        a = out[k]["a"]
        inr = lambda v, r: r[0] <= v <= r[1]
        if name == "a":                                 # x = a_i - a_(i-1)
            prev = a[-1] if a else 0
            return [x for x in range(-16, 17) if inr(prev + x, A_RANGE)]
        return [x for x in range(E_RANGE[0], E_RANGE[1] + 1) if inr(a[-1] + x, AE_RANGE)]

    def assign(vi, k):
        name, keys = var[vi]
        # candidates nearest a per-generator preference first, so that the generators spread over the range
        pref = (3 * k + 2 * vi) % 9 - 5
        for x in sorted(domain(k, name if name == "a" else "e"), key=lambda x: (abs(x - pref), x)):
            if not ok(k, keys, x):
                continue
            for key, sign in keys.items():
                hdr[k][key] = base[k][key] + sign * x
            if name == "a":
                out[k]["a"].append((out[k]["a"][-1] if out[k]["a"] else 0) + x)
            else:
                out[k]["e"][name[1:]] = x
            if k + 1 == len(SEEDS) or assign(vi, k + 1):
                return True
            for key in keys:
                del hdr[k][key]
            if name == "a":
                out[k]["a"].pop()
            else:
                del out[k]["e"][name[1:]]
        return False

    for vi in range(len(var)):
        assert assign(vi, 0), f"{cfg}: no exponents for {var[vi][0]}"
    return out


def rescaled_state_dict(sd, cfg, x):
    """State dict sd (weight-normed, checkpoint layout) rescaled by exponents x (the module docstring's a_i and e)."""
    h, n_st, n_k, n_dil = _hd(cfg)
    sd = {k: v.clone() for k, v in sd.items()}
    a = x["a"]                                         # a[0] = a_-1 (conv_pre's output), a[i + 1] = stage i's

    def scale(base, w, b):
        sd[base + ".weight_g"] *= 2.0 ** w
        if b is not None:
            sd[base + ".bias"] *= 2.0 ** b
    scale("conv_pre", a[0], a[0])
    for i in range(n_st):
        scale(f"ups.{i}", a[i + 1] - a[i], a[i + 1])
        for rb in range(i * n_k, (i + 1) * n_k):
            for d in range(n_dil):
                e = x["e"][(rb, d)]
                scale(f"resblocks.{rb}.convs1.{d}", e, a[i + 1] + e)
                scale(f"resblocks.{rb}.convs2.{d}", -e, a[i + 1])
    scale("conv_post", -a[n_st], None)
    return sd


_CACHE = {}


def exponents(cfg):
    if ("x", cfg) not in _CACHE:
        _CACHE[("x", cfg)] = _exponents(cfg)
    return _CACHE[("x", cfg)]


def seed_state_dicts(cfg):
    """The 8 seeds' state dicts, not rescaled (CPU), cached per config."""
    if ("seed", cfg) not in _CACHE:
        h = AttrDict(CFGS[cfg])
        _CACHE[("seed", cfg)] = [synth.hifigan_state_dict(h, seed=s) for s in SEEDS]
    return _CACHE[("seed", cfg)]


def state_dicts(cfg):
    """The 8 generators' state dicts (CPU, weight-normed), cached per config."""
    if ("sd", cfg) not in _CACHE:
        _CACHE[("sd", cfg)] = [rescaled_state_dict(sd, cfg, x) for sd, x in zip(seed_state_dicts(cfg), exponents(cfg))]
    return _CACHE[("sd", cfg)]


def check_pairwise(pks):
    """AssertionError unless, between every pair of packed generators, every tensor-core layer's header and tile bytes differ, and
    every other packed tensor (biases, b_post included, and the fp32 weights of the exact path) differs."""
    for a, b in itertools.combinations(range(len(pks)), 2):
        for k in pks[a]:
            if k.endswith("_tc"):
                assert header_exp(pks[a][k]) != header_exp(pks[b][k]), f"{k}: generators {a} and {b} share the header"
                assert not torch.equal(pks[a][k][packing.TC_HEADER_BYTES:], pks[b][k][packing.TC_HEADER_BYTES:]), \
                    f"{k}: generators {a} and {b} share the tiles"
            else:
                assert not torch.equal(pks[a][k], pks[b][k]), f"{k}: generators {a} and {b} share it"


def check_neighbours(pk, cfg):
    """AssertionError unless every ResBlock conv's header differs from those of its neighbouring slots within the generator."""
    _, n_st, n_k, n_dil = _hd(cfg)
    for k in pk:
        if k.startswith("rb.") and k.endswith("_tc"):
            for n in _neighbours(k[:-3], n_k, n_dil):
                assert header_exp(pk[k]) != header_exp(pk[n + "_tc"]), f"{k} and {n}_tc share the header"


def check_sane(sd, cfg, frames=48, seed=11):
    """One generator through the fp32 CPU oracle: finite, peak above 0.05 and under 1 % of the samples with |y| > 0.999."""
    from oracle import fs2_oracle as O
    y = O.hifigan_forward(sd, synth.make_mel(1, frames, seed=seed), **oracle_kwargs(cfg))
    assert torch.isfinite(y).all()
    peak, sat = float(y.abs().max()), float((y.abs() > 0.999).double().mean())
    assert peak > 0.05 and sat < 0.01, (peak, sat)
    return peak, sat


def oracle_kwargs(cfg):
    h = AttrDict(CFGS[cfg])
    return dict(upsample_rates=tuple(h.upsample_rates), upsample_kernel_sizes=tuple(h.upsample_kernel_sizes),
                resblock_kernel_sizes=tuple(h.resblock_kernel_sizes), resblock_dilation_sizes=tuple(map(tuple, h.resblock_dilation_sizes)))


# ---------------------------------------------------------------- the pool's launches and their work lists
F_FAR = 1 << 16                                        # a window origin no utterance end clips (the unclipped plan of the pool's call)


def model_of(cfg, policy):
    """The fs2_vocoder_model shape fields and masks a generator of cfg packs under policy (no weights: the plans read no pointer)."""
    g = _policy_generator(cfg, policy)
    h = AttrDict(CFGS[cfg])
    m = L.VocoderModel()
    m.n_mel, m.c0 = 80, h.upsample_initial_channel
    m.n_stages, m.n_kernels, m.n_dil = len(h.upsample_rates), len(h.resblock_kernel_sizes), len(h.resblock_dilation_sizes[0])
    for i, (u, k) in enumerate(zip(h.upsample_rates, h.upsample_kernel_sizes)):
        m.rates[i], m.up_k[i] = u, k
    for j, (k, dils) in enumerate(zip(h.resblock_kernel_sizes, h.resblock_dilation_sizes)):
        m.rb_k[j] = k
        for d, dv in enumerate(dils):
            m.rb_dil[j][d] = dv
    m.f8_mask, m.fused_mask, m.pair_mask, m.pair_kmax = g.effective_masks()
    return m, bool(g.use_tensor_cores)


def pool_launches(m, chunk):
    """A pool step's launches (fs2_vocoder_window_plan of an unclipped window of `chunk` frames), rows relative to the window."""
    out = L.vocoder_window_plan(m, 1 << 20, F_FAR, F_FAR + chunk)
    for l in out:
        l.y0, l.y1, l.x0, l.x1 = (v - F_FAR * l.scale for v in (l.y0, l.y1, l.x0, l.x1))
    return out


def resstack_tile(m, l):
    """(H, TILE) of a fused launch (VW_RB_GROUP / VW_RB_PAIR), as resstack_plan computes them (fs2_resstack_plan only serves 8 to 64
    channels, so the 128-channel pairs are planned here; tests/test_stream_multi_plans_cpu.py checks this against fs2_resstack_plan)."""
    C = m.c0 >> (l.stage + 1)
    Cm = max(C, 16)
    if l.layer == L.VW_RB_PAIR:
        js, d0, d1 = [l.j], l.d, l.d + 1
    elif l.j < 0:
        js, d0, d1 = range(m.n_kernels), 0, m.n_dil
    else:
        run = next(r for r in L.vocoder_resblock_runs(m, l.stage) if r.j == l.j and r.d0 == l.d)
        js, d0, d1 = [l.j], run.d0, run.d1
    H = max(sum((m.rb_k[j] - 1) * m.rb_dil[j][d] // 2 + (m.rb_k[j] - 1) // 2 for d in range(d0, d1)) for j in js)
    H = (H + 3) & ~3
    MT = 128 // Cm
    for hc in range(H, H + 33, 4):
        tile = MT * 128 - 2 * hc
        if tile < 64:
            break
        if any(tile % r == 0 and tile // r <= 12 for r in range(256, 7, -8)):
            return hc, tile
    raise AssertionError("no output box split")


def window_items(lens, f0s, scale, y0, yend, tile, blocks=1):
    """The stream of each work item of a windowed launch, in the kernels' order (WindowList: block group, stream, live tile): stream b's
    live rows are [-f0s[b] * scale, (lens[b] - f0s[b]) * scale), its tiles `tile` rows from the window's first row y0."""
    seq = []
    for _ in range(blocks):
        for b, (n, f0) in enumerate(zip(lens, f0s)):
            lo, hi = -f0 * scale, (max(n, 0) - f0) * scale
            first = max(0, lo - y0) // tile
            seq += [b] * max(0, max(0, min(hi, yend) - y0 + tile - 1) // tile - first)
    return seq


def cta_items(seq, grid):
    """Each persistent CTA's work items (item c, c + grid, ...) as their streams."""
    return [seq[c::grid] for c in range(grid)]


def switches(seq, grid):
    """Consecutive work items of one CTA (item i, i + grid) whose streams have different generators."""
    return sum(gen_of(seq[i]) != gen_of(seq[i + grid]) for i in range(len(seq) - grid))


def launch_kernels(m, tc, B, lens, f0s, chunk, sms):
    """Every launch of a pool step of B added streams (lengths lens, first frames f0s): a dict per launch with its name, kernel, plan and
    work-list facts.  kernel: 'conv_tc' (grid, NG, units per CTA, stream per item), 'conv_simt' (BM, BN), 'resstack' (width, run, grid,
    stream per item) or 'conv_post' (C)."""
    launches = pool_launches(m, chunk)
    convs = dict(zip([i for i, l in enumerate(launches) if l.layer <= L.VW_RB_CONV2], vocoder_convs(m, B, launches)))
    out = []
    for i, l in enumerate(launches):
        rows = l.y1 - l.y0
        if l.layer == L.VW_CONV_POST:
            out.append(dict(name="conv_post", kernel="conv_post", C=m.c0 >> m.n_stages))
            continue
        if l.layer in (L.VW_RB_GROUP, L.VW_RB_PAIR):
            C = m.c0 >> (l.stage + 1)
            _, tile = resstack_tile(m, l)
            grid = min(B * -(-rows // tile), sms)
            seq = window_items(lens, f0s, l.scale, l.y0, l.y1, tile)
            rb = l.stage * m.n_kernels + max(l.j, 0)
            out.append(dict(name=f"{'group' if l.layer == L.VW_RB_GROUP else 'pair'} stage {l.stage} rb {rb} d0 {max(l.d, 0)}",
                            kernel="resstack", width=C, j=l.j, d0=max(l.d, 0), grid=grid, seq=seq))
            continue
        name, a = convs[i]
        if tc and _on_tensor_cores(a):
            p = G.plan_args(a, sms)
            groups = a.N // p["NB"] // p["NG"]
            seq = window_items(lens, f0s, l.scale, l.y0, l.y1, 128, groups)
            units = max(len(s) for s in cta_items(seq, p["grid"])) * p["NG"]
            out.append(dict(name=name, kernel="conv_tc", NG=p["NG"], grid=p["grid"], units=units, seq=seq))
        else:
            sp = L.ConvSimtPlan()
            assert L.lib().fs2_conv_simt_plan(ctypes.byref(a), sms, ctypes.byref(sp)) == 0, name
            out.append(dict(name=name, kernel="conv_simt", BM=sp.BM, BN=sp.BN))
    return out


def _on_tensor_cores(a):
    """The conv runs on the tensor cores: its packed tiles exist (N % 16 == 0) and conv_tc_supported takes the shape."""
    out = L.ConvTcPlan()
    return a.N % 16 == 0 and L.lib().fs2_conv_tc_plan(ctypes.byref(a), 132, ctypes.byref(out)) == 0


# ---------------------------------------------------------------- the pools
CHUNK = 32


def pool_lens(n, seed=0):
    """n stream lengths in frames, 33 to 96 (two to three chunks), spread so that streams' live tiles differ."""
    return [33 + (b * 37 + seed * 11) % 64 for b in range(n)]


# (cfg, policy) -> the pool sizes its GPU test runs: all 8 generators, every stream added at tick 0 with pool_lens.  V1's 96 streams put
# the per-layer ResBlock convs of stages 0 and 1 at NG >= 2 and wrap the conv's slot ring; V2 needs 280 for ups 0's phase groups at NG >= 2
# (one 128-row tile per stream).  The exact policy runs pools of 3 and 24 streams too, for the 64-row tiles of small grids, and V2's
# 160 streams give conv_pre 64-row tiles at 128 columns.
POOLS = {("v1", "default"): (96,), ("v1", "exact"): (3, 24, 96), ("v1", "per_layer"): (96,), ("v1", "wide_pairs"): (96,),
         ("v2", "default"): (280,), ("v2", "exact"): (3, 24, 160), ("v2", "per_layer"): (280,), ("v2", "pairs"): (280,)}
