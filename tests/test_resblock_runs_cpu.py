"""CPU: the ResBlock run planner (fs2_vocoder_resblock_runs) -- how each fused stage is cut into fs2_resstack launches -- and the
windowed plan's invariants under those runs.  The GPU side (runs against the whole-group launch, bit for bit) is
tests/test_gpu_resblock_runs.py."""
import ctypes

import pytest

from fastspeech2_b200 import _lib as L
from tests.test_stream_vocoder_cpu import CONFIGS, _check_plan, _model


def _runs(m):
    return {i: L.vocoder_resblock_runs(m, i) for i in range(m.n_stages)}


def _plan_of(m, i, j, d0, d1, accumulate=0):
    """fs2_resstack_plan of ResBlock j's dilations [d0, d1) at stage i (j = -1: the whole group)."""
    js = range(m.n_kernels) if j < 0 else [j]
    a = L.ResstackArgs(B=16, N=1012 * 128, C=m.c0 >> (i + 1), n_kernels=len(js), n_dil=d1 - d0, accumulate=accumulate)
    for jj, src in enumerate(js):
        a.k[jj] = m.rb_k[src]
        for d in range(d0, d1):
            a.dil[jj][d - d0] = m.rb_dil[src][d]
    p = L.ResstackPlan()
    assert L.lib().fs2_resstack_plan(ctypes.byref(a), 132, ctypes.byref(p)) == 0
    return p


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_runs_cover_every_resblock_in_order_within_the_slab(cfg):
    m, _ = _model(CONFIGS[cfg])
    for i, runs in _runs(m).items():
        if not (m.fused_mask >> i) & 1:
            assert runs == []
            continue
        assert runs
        if runs[0].j < 0:
            assert len(runs) == 1 and (runs[0].d0, runs[0].d1) == (0, m.n_dil)
        else:                                          # ResBlock after ResBlock, each one's dilations in consecutive runs
            assert [r.j for r in runs] == sorted(r.j for r in runs) and {r.j for r in runs} == set(range(m.n_kernels))
            for j in range(m.n_kernels):
                mine = [r for r in runs if r.j == j]
                assert mine[0].d0 == 0 and mine[-1].d1 == m.n_dil and all(a.d1 == b.d0 for a, b in zip(mine, mine[1:]))
        for r in runs:
            p = _plan_of(m, i, r.j, r.d0, r.d1)
            assert (r.H, r.TILE, r.slab) == (p.H, p.TILE, p.MT * 128)
            assert r.TILE + 2 * r.H == r.slab and r.TILE >= 64 and r.cost > 0
            # the halo holds the run's receptive radius
            js = range(m.n_kernels) if r.j < 0 else [r.j]
            reach = max(sum((m.rb_k[j] - 1) * m.rb_dil[j][d] // 2 + (m.rb_k[j] - 1) // 2 for d in range(r.d0, r.d1)) for j in js)
            assert reach <= r.H


def test_v1_cuts_long_reach_resblocks():
    """V1 (kernels 3, 7, 11, dilations 1, 3, 5): the 64-channel stage keeps k = 3 whole, runs k = 7 as {1, 3} {5} and k = 11 one
    dilation per launch; the 32-channel stage splits only k = 11.  Recompute factors slab / TILE as planned."""
    m, _ = _model(CONFIGS["v1"])
    runs = _runs(m)
    assert [(r.j, r.d0, r.d1) for r in runs[2]] == [(0, 0, 3), (1, 0, 2), (1, 2, 3), (2, 0, 1), (2, 1, 2), (2, 2, 3)]
    assert [(r.H, r.TILE) for r in runs[2]] == [(12, 232), (20, 216), (20, 216), (12, 232), (20, 216), (32, 192)]
    assert [(r.j, r.d0, r.d1) for r in runs[3]] == [(0, 0, 3), (1, 0, 3), (2, 0, 2), (2, 2, 3)]
    # today's alternative, the whole group, recomputes 1.88x at 64 channels: every run here does less
    whole = _plan_of(m, 2, -1, 0, 3)
    assert (whole.H, whole.TILE) == (60, 136)
    assert all(r.slab / r.TILE < 1.34 < whole.MT * 128 / whole.TILE for r in runs[2])


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_window_plan_has_one_launch_per_run(cfg):
    m, _ = _model(CONFIGS[cfg])
    runs = _runs(m)
    P = L.vocoder_window_plan(m, 300, 100, 164)
    for i in range(m.n_stages):
        got = [(l.j, l.d) for l in P if l.stage == i and l.layer == L.VW_RB_GROUP]
        assert got == [(r.j, -1 if r.j < 0 else r.d0) for r in runs[i]]


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_window_plan_invariants_under_runs(cfg):
    """Reads inside producers, consecutive windows tile the waveform, streamed work within 10 % of offline."""
    m, up = _model(CONFIGS[cfg])
    for T, f0, f1 in ((1, 0, 1), (40, 0, 16), (101, 33, 54), (101, 95, 140), (1012, 500, 564)):
        _check_plan(m, up, T, f0, f1)
    T = 1012
    edges = [L.vocoder_window_plan(m, T, f0, f0 + 64)[-1] for f0 in range(0, T, 64)]
    assert edges[0].y0 == 0 and edges[-1].y1 == T * up and all(a.y1 == b.y0 for a, b in zip(edges, edges[1:]))
    offline = sum(l.flops for l in L.vocoder_window_plan(m, T, 0, T))
    streamed = sum(l.flops for f0 in range(0, T, 64) for l in L.vocoder_window_plan(m, T, f0, f0 + 64))
    assert streamed / offline <= 1.10


def test_bad_queries_are_refused():
    m, _ = _model(CONFIGS["v1"])
    h = L.lib()
    assert h.fs2_vocoder_resblock_runs(ctypes.byref(m), -1, None, 0) == -1
    assert h.fs2_vocoder_resblock_runs(ctypes.byref(m), m.n_stages, None, 0) == -1
    assert h.fs2_vocoder_resblock_runs(ctypes.byref(m), 2, None, -1) == -1
    assert h.fs2_vocoder_resblock_runs(ctypes.byref(m), 0, None, 0) == 0   # the 256-channel stage is not fused
    out = (L.ResblockRun * 2)()
    n = h.fs2_vocoder_resblock_runs(ctypes.byref(m), 2, out, 2)
    assert n == 6 and (out[0].j, out[1].j) == (0, 1)


def test_wide_pairs_plan_the_128_channel_stage():
    """pair_mask bit 8 + i (Generator.wide_pairs): V1's 128-channel stage runs its k = 3 pairs as fs2_resstack launches, widened by
    their reach in a window, and its k = 7 / 11 convs per layer; the public fs2_resstack still refuses 128 channels, and a fused_mask
    bit on that stage is refused."""
    m, up = _model(CONFIGS["v1"])
    m.pair_mask |= 0b10 << 8
    m.f8_mask |= 0b100
    P = L.vocoder_window_plan(m, 300, 100, 164)
    s1 = [l for l in P if l.stage == 1 and l.layer in (L.VW_RB_PAIR, L.VW_RB_CONV1, L.VW_RB_CONV2)]
    assert [(l.j, l.d) for l in s1 if l.layer == L.VW_RB_PAIR] == [(0, 0), (0, 1), (0, 2)]
    assert all(l.j > 0 for l in s1 if l.layer != L.VW_RB_PAIR)
    for T, f0, f1 in ((1, 0, 1), (101, 33, 54), (1012, 500, 564)):
        _check_plan(m, up, T, f0, f1)
    a = L.ResstackArgs(B=1, N=1000, C=128, n_kernels=1, n_dil=1)
    a.k[0], a.dil[0][0] = 3, 1
    assert L.lib().fs2_resstack_plan(ctypes.byref(a), 132, ctypes.byref(L.ResstackPlan())) == -2
    m.fused_mask |= 0b10
    assert L.lib().fs2_vocoder_resblock_runs(ctypes.byref(m), 1, None, 0) == -2


def test_wide_kernel_and_its_windowed_entry_point_are_pipelined_without_stack():
    """The 128-channel entry points (resstack_wide_kernel, _streams_): queued wgmma groups, no stack, no local memory."""
    import re
    import subprocess
    from tests.test_sass_pipeline import LIB, _cuobjdump
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    sass, name = {}, None
    for line in subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if "resstack_wide" in m.group(1) else None
            if name:
                sass[name] = []
        elif name:
            sass[name].append(line)
    usage, name = {}, None
    for line in subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1) if "resstack_wide" in m.group(1) else None
        elif name and "REG:" in line:
            usage[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            name = None
    assert len(sass) == 3 and set(sass) == set(usage), sorted(sass)
    for f, lines in sass.items():
        text = "\n".join(lines)
        mmas = len(re.findall(r"\b[HQ]GMMA\.", text))
        full_waits = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", text))
        assert mmas > 0 and full_waits * 4 <= mmas, (f, mmas, full_waits)
        assert usage[f]["STACK"] == 0 and usage[f]["LOCAL"] == 0, (f, usage[f])
