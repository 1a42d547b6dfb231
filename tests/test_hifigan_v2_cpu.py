"""HiFi-GAN V2 (configs.HIFIGAN_V2_CONFIG: stages of 64, 32, 16 and 8 channels) without a GPU: the module's keys against the reference
fixture (tests/golden/hifigan_v2.npz, oracle/gen_golden_hifigan_v2.py), the oracle against the reference's waveform, the fused
ResBlock kernel's launch plan at 16 and 8 channels, the Generator's default policy masks, and the narrow kernels' SASS."""
import ctypes
import json
import os
import re

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib, configs, packing, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from oracle import fs2_oracle as O
from tests import test_sass_pipeline as SP

GOLD = os.path.join(os.path.dirname(__file__), "golden", "hifigan_v2.npz")
V2 = AttrDict(configs.HIFIGAN_V2_CONFIG)
V1 = AttrDict(configs.HIFIGAN_CONFIG)
SHIPPED = ((3, 7, 11), ((1, 3, 5),) * 3)


def _fixture():
    return np.load(GOLD)


def test_state_dict_keys_match_reference_v2():
    z = _fixture()
    gen = Generator(V2)
    assert {k: list(v.shape) for k, v in gen.state_dict().items()} == json.loads(str(z["keys_weight_norm"]))
    gen.load_state_dict(synth.hifigan_state_dict(V2, seed=int(z["seed"])))
    gen.eval()
    gen.remove_weight_norm()
    assert {k: list(v.shape) for k, v in gen.state_dict().items()} == json.loads(str(z["keys_folded"]))


def test_oracle_reproduces_reference_v2():
    z = _fixture()
    threads = torch.get_num_threads()
    torch.set_num_threads(1)                  # the summation order the fixture was made with
    try:
        wav = O.hifigan_forward(synth.hifigan_state_dict(V2, seed=int(z["seed"])), torch.from_numpy(z["mel"]))
    finally:
        torch.set_num_threads(threads)
    assert wav.shape == z["wav"].shape
    assert (wav - torch.from_numpy(z["wav"])).abs().max() < 1e-6


def _rs_plan(C, N, ks=SHIPPED[0], dils=SHIPPED[1], B=16, lens=0):
    a = _lib.ResstackArgs(B=B, N=N, C=C, n_kernels=len(ks), n_dil=len(dils[0]), lens=lens, lens_scale=256 if lens else 0)
    for j, k in enumerate(ks):
        a.k[j] = k
        for d, dv in enumerate(dils[j]):
            a.dil[j][d] = dv
    out = _lib.ResstackPlan()
    rc = _lib.lib().fs2_resstack_plan(ctypes.byref(a), 132, ctypes.byref(out))
    return rc, _lib.fields(out)


@pytest.mark.parametrize("C", [16, 8])
def test_resstack_plan_narrow_widths(C):
    """16 and 8 channels: MT = 8 (MT * 16 = 128 accumulator columns, as for the wide widths), the slab is TILE + 2H = MT * 128 rows,
    the output boxes tile TILE, shared memory fits the SM; the grid comes from the padded shape whatever the lengths."""
    for ks, dils in [SHIPPED, ((3,), ((1,),)), ((11,), ((5,),)), ((3, 5), ((1, 2), (2, 6)))]:
        for N in (1, 50, 896, 897, 129536, 259072):
            rc, p = _rs_plan(C, N, ks, dils)
            assert rc == 0, (C, N, ks)
            assert p["MT"] == 8 and p["acc_regs"] == 128 and p["TPS"] == 8
            assert p["TILE"] + 2 * p["H"] == p["MT"] * 128
            assert p["H"] >= max(sum((k - 1) * d // 2 + (k - 1) // 2 for d in dj) for k, dj in zip(ks, dils))
            assert p["OBOX"] % 8 == 0 and p["OBOX"] * p["n_oboxes"] == p["TILE"] and p["n_oboxes"] <= 12
            assert p["smem"] <= 227 * 1024 and p["SB"] >= 2
            assert p["n_items"] == 16 * -(-N // p["TILE"]) and p["grid"] == min(p["n_items"], 132)
            assert _rs_plan(C, N, ks, dils, lens=0x1000)[1] == p
    # the shipped group: a 1024-row slab, H = 60 widened to whole 8-row boxes
    assert _rs_plan(C, 20000)[1]["TILE"] == 896


def test_resstack_plan_refuses_other_widths():
    for C in (24, 48, 4, 128):
        assert _rs_plan(C, 1000)[0] == -2, C
    for C in (8, 16):
        assert _rs_plan(C, 1000, (3,), ((33,),))[0] == -2       # reach beyond 32 rows


def test_default_masks_v1_unchanged_v2_fuses_every_stage():
    g1, g2 = Generator(V1), Generator(V2)
    assert (g1.f8_mask, g1.fused_mask, g1.pair_mask, g1.pair_kmax) == (0b11110, 0b1100, 0b0100, 3)
    assert g1.effective_masks() == (0b11110, 0b1100, 0, 3)
    assert g2.fused_mask == 0b1111
    assert g2.effective_masks() == (0b11110, 0b1111, 0, 3)
    # fusion never reaches a width fs2_resstack does not serve: V1's 256- and 128-channel stages
    g1.fused_mask = 0b1111
    assert g1.effective_masks()[1] == 0b1100
    g2.fused_mask, g2.pair_mask = 0, 0b1100
    assert g2.effective_masks() == (0b11110 | 0b11000, 0, 0b1100, 3)
    g2.use_tensor_cores = False
    assert g2.effective_masks() == (0, 0, 0, 0)


def test_pack_vocoder_pads_8_channel_tiles():
    """An 8-channel ResBlock conv in an f8 stage gets the 16 x 16 zero-padded tiles; in a stage without f8 it gets none."""
    gen = Generator(V2)
    f = lambda b: gen._folded(b).float()
    bias = lambda b: torch.zeros(1)
    pk = packing.pack_vocoder(f, bias, V2["upsample_rates"], 12, 3, f8_mask=0b11110)
    w = pk["rb.9.0.w1"]
    assert w.shape == (3, 8, 8)
    assert torch.equal(pk["rb.9.0.w1_tc"], packing.pack_conv_tc_pad16(w))
    wp = torch.zeros(3, 16, 16)
    wp[:, :8, :8] = w
    assert torch.equal(pk["rb.9.0.w1_tc"], packing.pack_conv_tc(wp, f8=True))
    assert packing.pack_conv_tc_pad16(torch.zeros(3, 16, 16)) is None
    pk0 = packing.pack_vocoder(f, bias, V2["upsample_rates"], 12, 3, f8_mask=0b01110)
    assert "rb.9.0.w1_tc" not in pk0 and "rb.6.0.w1_tc" in pk0


NARROW = "resstack_narrow_kernel"


@pytest.fixture(scope="module")
def narrow_sass():
    funcs, name = {}, None
    for line in SP._dump("-sass").splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if NARROW in m.group(1) else None
            if name:
                funcs[name] = []
        elif name:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


def test_narrow_kernels_in_sass_pipelined_without_spills(narrow_sass):
    """Both widths, padded and ragged; their wgmma pipelines are not serialised (the rule of tests/test_sass_pipeline.py), and they
    do not spill, except the ragged 16-channel kernel: a 16-byte stack frame for per-item state (the shared-memory barrier pointer,
    the ragged cursor, the fragment row base) that it stores once per work item and reloads at the item and kernel-size loop heads,
    outside the MMA and epilogue loops.  Its frame size is pinned so that any growth shows here."""
    assert len(narrow_sass) == 4 and all(SP._kernel(n) is None for n in narrow_sass)
    for name, text in narrow_sass.items():
        mmas = len(re.findall(r"\b[HQ]GMMA\.", text))
        full_waits = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", text))
        assert mmas > 0 and full_waits * 4 <= mmas, (name, mmas, full_waits)
    usage, name = {}, None
    for line in SP._dump("-res-usage").splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1) if NARROW in m.group(1) else None
        elif name and "REG:" in line:
            usage[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            name = None
    assert set(usage) == set(narrow_sass)
    for name, r in usage.items():
        frame = 16 if "ILi16ELb1E" in name else 0
        assert r["LOCAL"] == 0 and r["STACK"] <= frame, (name, r)
