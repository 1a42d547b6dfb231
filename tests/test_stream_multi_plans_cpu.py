"""CPU: the generators of tests/generator_cases.py differ where the multi-generator pool's kernels look, and the pools that
tests/test_gpu_stream_multi_plans.py runs reach the plans large pools pick, on 132 SMs (H100 SXM) and 114 SMs (H100 PCIe).

Every pool is planned as its first step runs it: all streams added at tick 0, each at its first frame.  A work list is derived from the
window rows of each launch the way WindowList orders items (channel-block group, stream, live tile), and a persistent CTA runs items
c, c + grid, ...; a pool that stops reaching a listed plan shape fails here, naming the layer."""
import ctypes
import itertools

import pytest
import torch

from fastspeech2_b200 import _lib as L, synth
from fastspeech2_b200.hifigan import AttrDict
from oracle import fs2_oracle as O
from tests import generator_cases as GC

SMS = (132, 114)


# ---------------------------------------------------------------- the fixture
@pytest.fixture(scope="module", params=sorted(GC.CFGS))
def cfg(request):
    return request.param


@pytest.fixture(scope="module")
def packs(cfg):
    """Each generator packed as the default policy and (V1) wide_pairs pack it."""
    sds = GC.state_dicts(cfg)
    out = {"default": [GC.pack(sd, cfg) for sd in sds]}
    if cfg == "v1":
        out["wide_pairs"] = [GC.pack(sd, cfg, "wide_pairs") for sd in sds]
    return out


def test_every_header_tile_bias_and_weight_differs_between_every_pair_of_generators(cfg, packs):
    for policy, pks in packs.items():
        tc = [k for k in pks[0] if k.endswith("_tc")]
        # every tensor-core layer the pool runs: conv_pre, the phase groups, every ResBlock conv (V2's 8-channel stage as pad16 tiles,
        # V1's wide pairs at 128 columns)
        want = 1 + 2 * (4 if cfg == "v1" else 3) + 2 * 12 * 3
        assert len(tc) == want, (policy, len(tc))
        if cfg == "v2":
            assert pks[0]["rb.9.0.w1_tc"].numel() == 128 + 3 * 64 * 16      # the 8-channel stage: f8 tiles zero-padded to 16 x 16
        if policy == "wide_pairs":
            assert pks[0]["rb.3.0.w1_tc"].numel() == 128 + 3 * 8 * 64 * 128
        GC.check_pairwise(pks)


def test_every_resblock_header_differs_from_its_neighbouring_slots(cfg, packs):
    for pk in packs["default"]:
        GC.check_neighbours(pk, cfg)


def test_scales_stay_in_range_and_keep_each_generators_function(cfg):
    """Every rescaling exponent within its range, and each rescaled generator's fp64 oracle output equal to its seed's to fp64 rounding."""
    _, n_st, n_k, _ = GC._hd(cfg)
    mel = synth.make_mel(1, 12, seed=5)
    kw = GC.oracle_kwargs(cfg)
    for k, (x, sd, seed_sd) in enumerate(zip(GC.exponents(cfg), GC.state_dicts(cfg), GC.seed_state_dicts(cfg))):
        assert len(x["a"]) == n_st + 1 and all(GC.A_RANGE[0] <= a <= GC.A_RANGE[1] for a in x["a"]), (k, x["a"])
        for (rb, d), e in x["e"].items():
            assert GC.E_RANGE[0] <= e <= GC.E_RANGE[1] and GC.AE_RANGE[0] <= x["a"][rb // n_k + 1] + e <= GC.AE_RANGE[1], (k, rb, d, e)
        y = O.hifigan_forward(sd, mel, dtype=torch.float64, **kw)
        y0 = O.hifigan_forward(seed_sd, mel, dtype=torch.float64, **kw)
        assert (y - y0).abs().max().item() <= 1e-12, k


def test_every_generator_is_finite_and_not_saturated(cfg):
    for k, sd in enumerate(GC.state_dicts(cfg)):
        GC.check_sane(sd, cfg)


def test_the_old_pair_of_seeds_fails_the_header_check():
    """Seeds 3 and 11, not rescaled (the pools of tests/test_gpu_stream_multi.py), share headers: the check has teeth."""
    for cfg in GC.CFGS:
        h = AttrDict(GC.CFGS[cfg])
        pks = [GC.pack(synth.hifigan_state_dict(h, seed=s), cfg) for s in (3, 11)]
        with pytest.raises(AssertionError, match="share the header"):
            GC.check_pairwise(pks)
        same = sum(GC.header_exp(pks[0][k]) == GC.header_exp(pks[1][k]) for k in pks[0] if k.endswith("_tc"))
        assert same >= 40, (cfg, same)


# ---------------------------------------------------------------- the work lists
def test_window_items_follow_the_window_lists_order():
    """Two streams, 128-row tiles from window row -20: stream 0 at its first frame (rows below 0 are not live: its first tile starts at
    row -20 and is live), stream 1 in mid-utterance, stream 2 past its end; two block groups repeat the streams."""
    seq = GC.window_items([10, 100, 3], [0, 40, 8], 64, -20, 64 * 32 + 20, 128, blocks=2)
    per = [1 + (640 + 20 - 1) // 128, -(-(64 * 32 + 40) // 128), 0]
    assert seq == ([0] * per[0] + [1] * per[1]) * 2
    assert GC.cta_items(list(range(7)), 3) == [[0, 3, 6], [1, 4], [2, 5]]
    assert [GC.gen_of(b) for b in range(8)] == [3, 0, 5, 2, 7, 4, 1, 6]


def test_resstack_tiles_match_the_planner():
    """generator_cases.resstack_tile against fs2_resstack_plan (8 to 64 channels) and fs2_vocoder_resblock_runs."""
    for cfg, policy in GC.CFG_POLICIES:
        m, _ = GC.model_of(cfg, policy)
        runs = {i: {(r.j, r.d0): r for r in L.vocoder_resblock_runs(m, i)} for i in range(m.n_stages)}
        for l in GC.pool_launches(m, GC.CHUNK):
            if l.layer not in (L.VW_RB_GROUP, L.VW_RB_PAIR):
                continue
            H, tile = GC.resstack_tile(m, l)
            C = m.c0 >> (l.stage + 1)
            if l.layer == L.VW_RB_GROUP:
                r = runs[l.stage][(l.j, l.d)]
                assert (r.H, r.TILE) == (H, tile), (cfg, policy, l.stage, l.j, l.d)
            if C <= 64:
                a = L.ResstackArgs(B=3, N=l.y1 - l.y0, C=C, n_kernels=1, n_dil=1)
                a.k[0], a.dil[0][0] = m.rb_k[l.j], m.rb_dil[l.j][l.d]
                if l.layer == L.VW_RB_GROUP:
                    r = runs[l.stage][(l.j, l.d)]
                    a.n_dil = r.d1 - r.d0
                    for d in range(r.d0, r.d1):
                        a.dil[0][d - r.d0] = m.rb_dil[l.j][d]
                p = L.ResstackPlan()
                assert L.lib().fs2_resstack_plan(ctypes.byref(a), 132, ctypes.byref(p)) == 0
                assert (p.H, p.TILE) == (H, tile), (cfg, policy, l.stage, l.j, l.d)


def _pool_kernels(cfg, policy, sms):
    m, tc = GC.model_of(cfg, policy)
    out = []
    for n in GC.POOLS[(cfg, policy)]:
        out += [dict(k, n=n) for k in GC.launch_kernels(m, tc, n, GC.pool_lens(n), [0] * n, GC.CHUNK, sms)]
    return out


def _report(ks):
    for k in ks:
        if k["kernel"] == "conv_tc":
            print(f"  n={k['n']:3d} conv_tc  {k['name']:28s} NG={k['NG']} grid={k['grid']} units/CTA={k['units']} "
                  f"switches={GC.switches(k['seq'], k['grid'])}")
        elif k["kernel"] == "resstack":
            print(f"  n={k['n']:3d} resstack {k['name']:28s} C={k['width']} grid={k['grid']} items={len(k['seq'])} "
                  f"switches={GC.switches(k['seq'], k['grid'])}")


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("cfg_policy", GC.CFG_POLICIES, ids=[f"{c}-{p}" for c, p in GC.CFG_POLICIES])
def test_pools_reach_the_listed_plans(cfg_policy, sms):
    cfg, policy = cfg_policy
    ks = _pool_kernels(cfg, policy, sms)
    print(cfg, policy, sms)
    _report(ks)
    tc = [k for k in ks if k["kernel"] == "conv_tc"]
    if policy == "exact":
        assert not tc and not any(k["kernel"] == "resstack" for k in ks)
    else:
        # the tensor-core conv's multi mode with channel-block groups
        if cfg == "v2":
            for g in "ab":
                assert any(k["name"] == f"ups.0.{g}" and k["NG"] >= 2 for k in tc), f"ups.0.{g} never at NG >= 2"
        else:
            assert any(k["name"].startswith("resblocks.") and k["NG"] >= 2 for k in tc), "no per-layer ResBlock conv at NG >= 2"
        # a CTA with more units than the slot ring, whose consecutive items change generator
        wrap = [k["name"] for k in tc if k["units"] > GC.G.SLOTS and any(
            len(s) * k["NG"] > GC.G.SLOTS and any(GC.gen_of(x) != GC.gen_of(y) for x, y in zip(s, s[1:]))
            for s in GC.cta_items(k["seq"], k["grid"]))]
        assert wrap, "no conv_tc launch wraps the slot ring across generators"
    # every fused launch: some CTA runs consecutive items of different generators
    for k in ks:
        if k["kernel"] == "resstack":
            assert len(k["seq"]) > k["grid"] and GC.switches(k["seq"], k["grid"]) > 0, (k["n"], k["name"])
    # conv_post: the register-resident C = 32 kernel for V1, the generic one for V2
    C = {k["C"] for k in ks if k["kernel"] == "conv_post"}
    assert C == ({32} if cfg == "v1" else {8}), C


@pytest.mark.parametrize("sms", SMS)
def test_fused_widths_and_dilation_runs_are_covered(sms):
    """Across the policies of a config, the fused launches cover every width fs2_resstack runs in it, each with a launch whose first
    dilation is above 0 (the slot d0 + d), with consecutive items of different generators on some CTA."""
    for cfg, widths in (("v1", {128, 64, 32}), ("v2", {64, 32, 16, 8})):
        seen, d0 = set(), set()
        for c, policy in GC.CFG_POLICIES:
            if c != cfg:
                continue
            for k in _pool_kernels(cfg, policy, sms):
                if k["kernel"] == "resstack" and GC.switches(k["seq"], k["grid"]) > 0:
                    seen.add(k["width"])
                    if k["d0"] > 0:
                        d0.add(k["width"])
        assert seen == widths and d0 == widths, (cfg, seen, d0)


def _simt_universe(cfg, sms):
    """Every (BM, BN) fs2_conv_simt_plan gives the exact policy's window launches, pools of 1 to 1024 streams."""
    m, _ = GC.model_of(cfg, "exact")
    out = set()
    for n in (1, 2, 3, 4, 6, 8, 12, 16, 24, 32, 48, 64, 96, 128, 192, 256, 384, 512, 1024):
        out |= {(k["BM"], k["BN"]) for k in GC.launch_kernels(m, False, n, [n] * n, [0] * n, GC.CHUNK, sms) if k["kernel"] == "conv_simt"}
    return out


@pytest.mark.parametrize("sms", SMS)
def test_exact_pools_reach_every_simt_tile(sms):
    for cfg in GC.CFGS:
        got = {(k["BM"], k["BN"]) for k in _pool_kernels(cfg, "exact", sms) if k["kernel"] == "conv_simt"}
        want = _simt_universe(cfg, sms)
        assert {bm for bm, _ in want} == {64, 128}
        assert got == want, (cfg, sorted(want - got))


def test_gen_of_uses_every_generator_in_every_pool():
    for ns in GC.POOLS.values():
        assert {GC.gen_of(b) for b in range(max(ns))} == set(range(GC.MAX_GENERATORS))
    assert all(33 <= v <= 96 for v in GC.pool_lens(280))
    assert len(list(itertools.chain(*GC.POOLS.values()))) <= 14
