"""CPU: a census of the shipped models' tensor-core convs planned with channel-block groups (NG > 1), and the case table of
tests/conv_group_cases.py that the GPU tests run.

Every FastSpeech2 and HiFi-GAN V1 / V2 conv that runs on the tensor cores is planned through fs2_conv_tc_plan at 132 SMs (H100 SXM)
and 114 SMs (H100 PCIe), offline at B in {1, 16, 64, 512} x {1012, 2006} frames and in stream-pool windows of 64 and 512 streams x 32
frames.  Each one planned at NG > 1 must have a case of the table with its format, NB, block count, NG, K-blocks and taps per weight
stage: a planner change that sends a shipped layer into an untested group shape fails here, naming the layer."""
import ctypes

import pytest

from fastspeech2_b200 import _lib as L, configs
from tests import conv_group_cases as G
from tests.test_stream_vocoder_cpu import _model

SMS = (132, 114)
OFFLINE = [(B, T) for B in (1, 16, 64, 512) for T in (1012, 2006)]
POOLS = [(64, 32), (512, 32)]
F8, SPLIT3 = L.TC_VARIANT_F8, 0
SEG = L.TC_VARIANT_NB64 | L.TC_VARIANT_SEGMENTED


def _args(B, T, Cin, N, taps, dil=1, res=False, acc=False, variant=F8, in_act=L.ACT_NONE):
    return L.Conv1dArgs(x=0x1000, x_batch_stride=T * Cin, x_row_stride=Cin, B=B, T=T, Cin=Cin, w=0x1000, N=N, taps=taps, dilation=dil,
                        pad_left=(taps - 1) * dil // 2, w_tc=0x1000, y=0x1000, y_batch_stride=T * N, y_row_stride=N, alpha=1.0,
                        res=0x2000 if res else 0, res_batch_stride=T * N if res else 0, res_row_stride=N if res else 0,
                        accumulate=int(acc), tc_variant=variant, in_act=in_act, in_slope=0.1)


def _plan_or_none(a, sms):
    """The plan, or None for a shape the tensor-core kernel does not take (the layer then runs on the exact kernel)."""
    out = L.ConvTcPlan()
    rc = L.lib().fs2_conv_tc_plan(ctypes.byref(a), sms, ctypes.byref(out))
    return L.fields(out) if rc == 0 else None


def fs2_convs(B, T):
    """FastSpeech2's tensor-core convs at B x T rows, in the default tc_mask formats: (name, args).  The encoder and the variance
    predictors run K-segmented; the decoder's FFT convs, mel_linear and the PostNet in the f16 + f8 format."""
    D, F, k1 = 256, 1024, 9
    out = []
    for part, v in (("encoder", SEG), ("decoder", F8)):
        out += [(f"{part}.qkv", _args(B, T, D, 3 * D, 1, variant=v)), (f"{part}.proj", _args(B, T, D, D, 1, res=True, variant=v)),
                (f"{part}.ffn.w_1", _args(B, T, D, F, k1, variant=v)), (f"{part}.ffn.w_2", _args(B, T, F, D, 1, res=True, variant=v))]
    out += [(f"predictor.conv{i}", _args(B, T, D, D, 3, variant=SEG)) for i in (1, 2)]
    out.append(("mel_linear", _args(B, T, D, 80, 1)))
    post = [(80, 512)] + [(512, 512)] * 3 + [(512, 80)]
    out += [(f"postnet.{i}", _args(B, T, ci, co, 5, res=i == 4)) for i, (ci, co) in enumerate(post)]
    return out


def vocoder_convs(m, B, launches):
    """The per-layer tensor-core convs among a vocoder window plan's launches: (name, args) at the launch's rows."""
    fmt = lambda i: F8 if m.f8_mask & (2 << i) else SPLIT3
    out = []
    for l in launches:
        rows, i = l.y1 - l.y0, l.stage
        if l.layer == L.VW_CONV_PRE:
            out.append(("conv_pre", _args(B, rows, 80, m.c0, 7, variant=F8 if m.f8_mask & 1 else SPLIT3)))
        elif l.layer in (L.VW_UP_A, L.VW_UP_B):
            C, u = m.c0 >> i, m.rates[i]
            out.append((f"ups.{i}.{'ab'[l.layer - L.VW_UP_A]}", _args(B, rows, C, u // 2 * (C // 2), 2, variant=fmt(i),
                                                                      in_act=L.ACT_LRELU)))
        elif l.layer in (L.VW_RB_CONV1, L.VW_RB_CONV2):
            C, k = m.c0 >> (i + 1), m.rb_k[l.j]
            two = l.layer == L.VW_RB_CONV2
            acc = two and l.d == m.n_dil - 1 and l.j > 0
            out.append((f"resblocks.{i * m.n_kernels + l.j}.convs{1 + two}.{l.d}",
                        _args(B, rows, C, C, k, 1 if two else m.rb_dil[l.j][l.d], res=two, acc=acc, variant=fmt(i), in_act=L.ACT_LRELU)))
    return out


def census(sms):
    """{(model, layer, shape): (fmt, NB, blocks, NG, K-blocks, TPS)} of every shipped conv planned at NG > 1 on sms SMs."""
    found = {}

    def add(model, shape, convs):
        for name, a in convs:
            p = _plan_or_none(a, sms)
            if p and p["NG"] > 1:
                fmt = "f8" if a.tc_variant & F8 else "split3"
                found[(model, name, shape)] = (fmt, p["NB"], a.N // p["NB"], p["NG"], a.Cin // 16, p["TPS"])

    for B, T in OFFLINE:
        add("fastspeech2", f"B={B} T={T}", fs2_convs(B, T))
    for cfg in ("v1", "v2"):
        m, _ = _model(configs.HIFIGAN_CONFIG if cfg == "v1" else configs.HIFIGAN_V2_CONFIG)
        for B, T in OFFLINE:
            add(f"hifigan_{cfg}", f"B={B} T={T}", vocoder_convs(m, B, L.vocoder_window_plan(m, T, 0, T)))
        for n, frames in POOLS:
            f0 = 1 << 16
            add(f"hifigan_{cfg}", f"pool {n} x {frames}", vocoder_convs(m, n, L.vocoder_window_plan(m, 1 << 20, f0, f0 + frames)))
    return found


def case_key(c, sms):
    p = G.plan(c, G.choose_batch(c, sms), sms)
    return (c["fmt"], p["NB"], c["N"] // p["NB"], p["NG"], c["Cin"] // 16, p["TPS"])


@pytest.mark.parametrize("sms", SMS)
def test_every_shipped_conv_planned_with_groups_has_a_case(sms):
    keys = {case_key(c, sms) for c in G.CASES}
    found = census(sms)
    for (model, name, shape), key in sorted(found.items()):
        print(f"{sms} SMs  {model:12s} {name:28s} {shape:16s} fmt={key[0]} NB={key[1]} blocks={key[2]} NG={key[3]} "
              f"K-blocks={key[4]} TPS={key[5]}")
    missing = {k: v for k, v in found.items() if v not in keys}
    assert not missing, missing
    # the layers the benchmark's shapes send into groups (FastSpeech2's PostNet conv 0, V1's conv_pre and 128-channel stage, V2's
    # first two upsample stages): the census must see them, or it is not planning what ships
    names = {(model, name.rsplit(".", 1)[0] if name.startswith("ups") else name) for model, name, _ in found}
    for want in (("fastspeech2", "postnet.0"), ("hifigan_v1", "conv_pre"), ("hifigan_v2", "ups.0"), ("hifigan_v2", "ups.1")):
        assert want in names, want
    assert any(model == "hifigan_v1" and name.startswith("resblocks.") for model, name, _ in found)


@pytest.mark.parametrize("sms", SMS)
def test_the_shape_chooser_hits_every_cases_group_size(sms):
    for c in G.CASES:
        B = G.choose_batch(c, sms)
        p = G.plan(c, B, sms)
        nblk = c["N"] // p["NB"]
        assert p["NG"] == c["NG"] and nblk % p["NG"] == 0, (c["name"], p)
        assert p["n_items"] // p["NG"] >= 4 * sms and (p["n_items"] // p["NG"]) % p["grid"], (c["name"], p)
        # every larger divisor of the block count leaves fewer than 4 waves
        assert all(p["n_items"] // ng < 4 * sms for ng in range(c["NG"] + 1, nblk + 1) if nblk % ng == 0), (c["name"], p)
        assert c["T"] % 128, c["name"]                 # partial tiles on every CTA
        assert B * c["T"] <= 200 * 512, c["name"]      # many short utterances: the fp64 check stays cheap


def _plan_classes(c, p):
    """The classes a case's plan itself shows: where its slab falls in the slab ring, the weight ring's depth, the slot ring's wrap."""
    kb, SA = c["Cin"] // 16, p["SA"]
    out = set()
    if SA % kb:
        out.add("slab_wraps")                          # item slabs start at i * kb mod SA: some cross the ring's end
    if 2 * kb <= SA:
        out.add("slab_next_resident")                  # the next item's slab fits beside this one's during its earlier passes
    if SA == kb < G.SA_MAX:
        out.add("sa==kb<8")
    if kb < SA < G.SA_MAX:
        out.add("kb<sa<8")
    if p["SB"] == 2:
        out.add("sb2")
    if -(-p["n_items"] // p["NG"] // p["grid"]) * p["NG"] > G.SLOTS:
        out.add("slots>16")
    if c["N"] // p["NB"] > p["NG"]:
        out.add("group>0")
    if (c["taps"] - 1) * c["dil"] >= 250:
        out.add("halo256")
    return out


@pytest.mark.parametrize("sms", SMS)
def test_the_table_covers_every_class(sms):
    derived = {"slab_wraps", "slab_next_resident", "sa==kb<8", "kb<sa<8", "sb2", "slots>16", "group>0", "halo256"}
    covered = set()
    for c in G.CASES:
        p = G.plan(c, G.choose_batch(c, sms), sms)
        got = _plan_classes(c, p)
        claimed = set(c["cls"]) & derived
        assert claimed <= got, (c["name"], claimed - got)   # a label must be what the plan does
        covered |= G.classes(c) | got
        if "group>0" in c["cls"]:
            assert "group>0" in got, c["name"]
    for ng in (2, 3, 4, 8):                            # each NG with a group index above 0
        assert any(c["NG"] == ng and c["N"] // G.nb_of(c["fmt"], c["N"]) > ng for c in G.CASES), ng
    assert G.REQUIRED_CLASSES <= covered, G.REQUIRED_CLASSES - covered
    assert 40 <= len(G.CASES) <= 60 and len({c["name"] for c in G.CASES}) == len(G.CASES)
