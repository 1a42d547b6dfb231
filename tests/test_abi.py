"""CPU: the C-ABI library builds/loads without a GPU and exports every symbol include/fs2b200.h declares."""
import ctypes
import os
import re

import pytest

from fastspeech2_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "fs2b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fs2_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_loads():
    path = build.build()
    assert os.path.exists(path)
    h = _lib.lib()
    assert h.fs2_abi_version() == _lib.ABI_VERSION
    assert b"sm_90a" in h.fs2_build_info()


def test_every_declared_symbol_is_exported_and_bound():
    names = _declared()
    assert len(names) >= 19
    h = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(h, n), f"{n} declared in fs2b200.h but not exported"
        assert n in _lib.EXPORTS, f"{n} has no ctypes binding"


def test_struct_sizes_match_the_header():
    h = _lib.lib()
    table = {0: _lib.Conv1dArgs, 1: _lib.LayerNormArgs, 2: _lib.AttentionArgs, 3: _lib.EmbedArgs, 4: _lib.RowBiasArgs,
             5: _lib.VarianceHeadArgs, 6: _lib.DurationsArgs, 7: _lib.LengthRegulateArgs, 8: _lib.ConvPostArgs,
             9: _lib.AcousticModel, 10: _lib.EncodeArgs, 11: _lib.DecodeArgs, 12: _lib.VocoderModel, 13: _lib.VocoderArgs, 14: _lib.ResstackArgs, 15: _lib.WavInt16Args,
             16: _lib.ConvTcPlan, 17: _lib.ConvSimtPlan, 18: _lib.ResstackPlan}
    for i, cls in table.items():
        assert h.fs2_struct_size(i) == ctypes.sizeof(cls), cls.__name__


def test_host_side_argument_checks_need_no_gpu():
    h = _lib.lib()
    assert h.fs2_conv1d(None, None) == -1                       # FS2_ERR_ARG
    a = _lib.Conv1dArgs(x=16, w=16, y=16, B=1, T=4, Cin=24, N=16, taps=1)
    assert h.fs2_conv1d(ctypes.byref(a), None) == -2             # Cin % 16 -> FS2_ERR_UNSUPPORTED
    m = _lib.AcousticModel(d_model=256, n_head=2, d_inner=1024, k1=9, k2=1, n_enc=4, n_dec=6, n_mel=80, vp_filter=256,
                           vp_kernel=3, n_postnet=5)
    for i, c in enumerate([512, 512, 512, 512, 80]):
        m.post_cout[i] = c
    need = h.fs2_decode_workspace_bytes(ctypes.byref(m), 16, 1024)
    assert need > 16 * 1024 * (256 * 4 + 768 + 1024) * 4
    assert h.fs2_encode_workspace_bytes(ctypes.byref(m), 0, 5) == 0
    r = _lib.ResstackArgs(x=0x10000, y=0x10000 + 64, B=1, N=100, C=32, n_kernels=1, n_dil=1)
    assert h.fs2_resstack(ctypes.byref(r), None) == -1           # overlapping x / y (the kernel re-reads halo rows of x)
    r.y = 0x10008
    assert h.fs2_resstack(ctypes.byref(r), None) == -1           # misaligned y
    for backend in (1, 3):                                       # attention backends are 0 (exact) and 2 (fused tensor-core kernel)
        at = _lib.AttentionArgs(qkv=0x1000, ctx=0x1000, B=1, T=4, H=2, Dh=128, scale=1.0, backend=backend)
        assert h.fs2_attention(ctypes.byref(at), None) == -1


def _plan(h, B, T, Cin, N, taps, dil=1, num_sms=132, x=0x1000, x_row_stride=None, tc_variant=0):
    a = _lib.Conv1dArgs(x=x, x_batch_stride=T * (x_row_stride or Cin), x_row_stride=x_row_stride or Cin, B=B, T=T, Cin=Cin, w=0x1000, N=N, taps=taps,
                        dilation=dil, pad_left=(taps - 1) * dil // 2, w_tc=0x1000, y=0x1000, y_batch_stride=T * N, y_row_stride=N, alpha=1.0,
                        tc_variant=tc_variant)
    out = _lib.ConvTcPlan()
    rc = h.fs2_conv_tc_plan(ctypes.byref(a), num_sms, ctypes.byref(out))
    return rc, _lib.fields(out)


def test_tensor_core_conv_launch_plan_respects_the_hardware_limits():
    """Host-side heuristics of the wgmma conv (work-item shape, ring depths, register / shared-memory budget) for every layer shape of
    both models at the BASELINE batch sizes, plus a sweep: no plan may exceed 227 KB of shared memory, 64 accumulator registers per
    consumer thread, the register-ring row capacity or the ring maxima, and the work items must cover the problem exactly."""
    h = _lib.lib()
    shapes = []
    for B, T in ((1, 7), (1, 1012), (16, 1012), (64, 2032)):
        shapes += [(B, T, 256, 768, 1, 1), (B, T, 256, 256, 1, 1), (B, T, 256, 1024, 9, 1), (B, T, 1024, 256, 1, 1), (B, T, 256, 80, 1, 1),
                   (B, T, 80, 512, 5, 1), (B, T, 512, 512, 5, 1), (B, T, 512, 80, 5, 1)]
        shapes += [(B, T, 128, 2048, 1, 1), (B, T, 2048, 128, 1, 1)]          # sweep: wide N, long C_in
        t, c = T, 512
        shapes.append((B, T, 80, 512, 7, 1))                                   # conv_pre
        for u in (8, 8, 2, 2):
            shapes.append((B, t, c, (u // 2) * (c // 2), 2, 1))                # one ConvTranspose phase group
            t, c = t * u, c // 2
            shapes += [(B, t, c, c, k, d) for k in (3, 7, 11) for d in (1, 3, 5)]
    for (B, T, Cin, N, k, d) in shapes:
        rc, p = _plan(h, B, T, Cin, N, k, d, num_sms=132)
        assert rc == 0, (B, T, Cin, N, k, d, rc)
        assert p["NB"] % 16 == 0 and 16 <= p["NB"] <= 128 and N % p["NB"] == 0
        assert p["TG"] == (2 if p["NB"] <= 64 else 1)
        assert p["acc_regs"] == p["TG"] * p["NB"] // 2 <= 64
        assert p["smem"] <= 227 * 1024
        assert 2 <= p["SA"] <= 8 and 2 <= p["SB"] <= 8 and 1 <= p["TPS"] <= k
        assert p["R"] % 8 == 4 and p["R"] >= 128 + (k - 1) * d
        assert p["R"] <= 3 * 256 // 2 + 7                                      # rows the transform warps' register ring can hold
        assert p["tiles_per_batch"] * 128 >= T > (p["tiles_per_batch"] - 1) * 128
        assert p["n_items"] == (N // p["NB"]) * B * p["tiles_per_batch"] and p["grid"] == min(p["n_items"], 132)
    # the packer and the kernel agree on the work-item width of both tile formats (F8 tiles: at most 64 channels)
    from fastspeech2_b200 import packing
    for n in range(0, 1100, 8):
        assert h.fs2_conv_tc_block(n) == packing.conv_tc_block(n) and h.fs2_conv_tc_block_f8(n) == packing.conv_tc_block(n, 64), n
        if n and n % 16 == 0:
            a = _lib.Conv1dArgs(x=0x1000, x_batch_stride=256 * 16, x_row_stride=16, B=1, T=256, Cin=16, w=0x1000, N=n, taps=1,
                                w_tc=0x1000, y=0x1000, y_batch_stride=256 * n, y_row_stride=n, alpha=1.0, tc_variant=_lib.TC_VARIANT_F8)
            out = _lib.ConvTcPlan()
            assert h.fs2_conv_tc_plan(ctypes.byref(a), 132, ctypes.byref(out)) == 0 and out.NB == h.fs2_conv_tc_block_f8(n) and out.TG == 2, n
    # ring depths per shape class: short kernels get the deepest slab ring, wide kernels share one weight stage between four taps
    assert _plan(h, 16, 64768, 128, 128, 3)[1]["SA"] == 5 and _plan(h, 16, 64768, 128, 128, 11, 5)[1]["TPS"] == 4
    # refused shapes: C_in % 16, N % 16, misaligned or oddly strided x, halo beyond the slab
    assert _plan(h, 1, 128, 24, 16, 1)[0] == -2 and _plan(h, 1, 128, 16, 24, 1)[0] == -2
    assert _plan(h, 1, 128, 16, 16, 1, x=0x1010)[0] == -2 and _plan(h, 1, 128, 16, 16, 1, x_row_stride=20)[0] == -2
    assert _plan(h, 1, 4096, 16, 16, 11, 30)[0] == -2


def _rs_plan(C, N, ks, dils, B=16):
    a = _lib.ResstackArgs(B=B, N=N, C=C, n_kernels=len(ks), n_dil=len(dils[0]))
    for j, k in enumerate(ks):
        a.k[j] = k
        for d, dv in enumerate(dils[j]):
            a.dil[j][d] = dv
    out = _lib.ResstackPlan()
    rc = _lib.lib().fs2_resstack_plan(ctypes.byref(a), 132, ctypes.byref(out))
    return rc, _lib.fields(out)


def test_gpu_case_tables_reach_every_tile_width_and_the_persistent_loop():
    """The GPU op tests (tests/test_gpu_ops.py) launch every work-item width the conv dispatcher instantiates in both tile formats, give
    every CTA of a 132-SM grid at least two work items (some cases four) in each format, sit at the limits of the conv halo and of the
    ResBlock kernel's reach, and put the ResBlock group at one tile +- 1 row.  Checked here, without a GPU, so that a later edit cannot
    quietly shrink those tables."""
    from fastspeech2_b200 import packing
    from tests import test_gpu_ops as G
    h = _lib.lib()
    # every NB: split3 {16, ..., 128}, f8 {16, 32, 48, 64}
    assert {packing.conv_tc_block(c[3]) for c in G.TC_CASES} == set(range(16, 129, 16))
    assert {packing.conv_tc_block(c[3], 64) for c in G.TC_CASES} == {16, 32, 48, 64}
    # the persistent loop: >= 2 work items per CTA at 132 SMs in every format, >= 4 in at least one case of each
    tables = {0: G.TC_PERSISTENT_CASES, _lib.TC_VARIANT_F8: G.TC_PERSISTENT_CASES,
              _lib.TC_VARIANT_NB64 | _lib.TC_VARIANT_SEGMENTED: [(B, T, Cin, N, taps, 1) for B, T, Cin, N, taps, *_ in G.SEG_PERSISTENT_CASES]}
    for variant, cases in tables.items():
        items = []
        for B, T, Cin, N, taps, dil, *_ in cases:
            rc, p = _plan(h, B, T, Cin, N, taps, dil, tc_variant=variant)
            assert rc == 0 and p["grid"] == 132, (variant, B, T, Cin, N)
            items.append(p["n_items"])
        assert min(items) >= 2 * 132 and max(items) >= 4 * 132, (variant, items)
    assert len(G.TC_PERSISTENT_CASES) >= 5 and len(G.SEG_PERSISTENT_CASES) >= 3
    assert all(c in G.TC_CASES for c in G.TC_PERSISTENT_CASES) and all(c in G.SEG_CASES for c in G.SEG_PERSISTENT_CASES)
    assert any(B * 2 * -(-T // 128) >= 2 * 132 for T, lens in G.ATT_BATCHED_CASES for B in [len(lens)])     # fused attention items
    # conv halo (taps - 1) * dilation: 256 is planned (both 2 x 256 and 3 x 128 are in the table), 257 is refused
    halos = {(c[4], c[5]) for c in G.TC_CASES if (c[4] - 1) * c[5] == 256}
    assert {(2, 256), (3, 128)} <= halos
    assert {c[6] for c in G.TC_CASES if (c[4] - 1) * c[5] == 256} >= {0, 128, 256}                 # pad_left 0, centred, = halo
    for taps, dil in halos:
        assert _plan(h, 2, 700, 32, 64, taps, dil)[0] == 0
    assert _plan(h, 2, 700, 32, 64, 2, 257)[0] == -2 and _plan(h, 2, 700, 32, 64, 3, 129)[0] == -2
    # ResBlock: the tile of the shipped group, and single pairs whose taps reach exactly 32 rows (33 is refused)
    ship_k, ship_d = (3, 7, 11), ((1, 3, 5),) * 3
    for C, tile in G.RESSTACK_TILE.items():
        assert _rs_plan(C, 1000, ship_k, ship_d)[1]["TILE"] == tile
        assert {N for _, N, c, k, d in G.RESSTACK_CASES if c == C and k == ship_k and d == ship_d} >= {1, tile - 1, tile + 1}
    reach32 = {(C, k) for C, k, dils, N in G.SINGLE_PAIR_CASES if max((k - 1) * d // 2 for d in dils) == 32}
    assert reach32 == {(C, k) for C in (32, 64) for k in (3, 5, 9)}
    for C, k in reach32:
        assert _rs_plan(C, 1000, (k,), ((64 // (k - 1),),))[0] == 0
    assert _rs_plan(32, 1000, (3,), ((33,),))[0] == -2


def test_gpu_case_tables_reach_every_exact_conv_tile():
    """The exact fp32 conv tests (tests/test_gpu_ops.py::test_conv1d, ::test_conv1d_ragged) reach, on a 132-SM device, all six (BM, BN)
    tiles of conv_simt_kernel, each with all four output activations, a partial row tile and a partial column tile; plus T = 1, one
    K-step, 11 dilated taps, pad_left 0 and off-centre, alpha / residual / accumulate, row_lens, strided views, LRELU input with slopes
    0 and 0.1, and ragged lengths 0, 1, BM - 1, BM, BM + 1 and T with lens_scale 1 and 8.  Checked here against fs2_conv_simt_plan."""
    from tests import test_gpu_ops as G
    seen = {}
    for case in G.CONV_CASES:
        case, opts = G._case_opts(case)
        B, T, Cin, N, taps, dil, pad, in_act, out_act = case[:9]
        bm, bn = G.simt_plan(B, T, Cin, N, taps)
        s = seen.setdefault((bm, bn), {"acts": set(), "T_tail": False, "N_tail": False})
        s["acts"].add(out_act)
        s["T_tail"] |= T % bm != 0
        s["N_tail"] |= N % bn != 0
    assert set(seen) == G.SIMT_TILES
    for tile, s in seen.items():
        assert s["acts"] == {0, 1, 2, 3} and s["T_tail"] and s["N_tail"], (tile, s)
    cases = [G._case_opts(c) for c in G.CONV_CASES]
    assert any(c[1] == 1 for c, _ in cases) and any(c[2] == 16 for c, _ in cases)
    assert any(c[4] == 11 and c[5] > 1 for c, _ in cases)
    pads = {"zero": any(c[6] == 0 and c[4] > 1 for c, _ in cases), "off_centre": any(c[6] not in (0, (c[4] - 1) * c[5] // 2) for c, _ in cases)}
    assert all(pads.values()), pads
    assert any(c[9] and c[10] != 1.0 and c[11] for c, _ in cases) and any(c[12] for c, _ in cases)
    assert any(o.get("strided") for _, o in cases)
    assert {o.get("in_slope", 0.1) for c, o in cases if c[7] == 3} == {0.0, 0.1}
    assert {G.simt_plan(*c[:5])[1] for c, _ in cases if c[3] % 4 == 0 and c[3] <= 32} == {32}     # GW = 2 stores
    # ragged: row counts 0, 1, BM - 1, BM, BM + 1, T in both row tiles (lens_scale 1), and lens_scale 8
    for bm in (64, 128):
        rows = set()
        for B, T, Cin, N, taps, *_, scale, xl in G.RAGGED_CONV_CASES:
            if G.simt_plan(B, T, Cin, N, taps)[0] == bm and scale == 1:
                rows |= {min(l * scale, T) for l in xl} | ({"T"} if T in xl else set())
        assert {0, 1, bm - 1, bm, bm + 1, "T"} <= rows, (bm, rows)
    assert {c[9] for c in G.RAGGED_CONV_CASES} == {1, 8}
    assert any(l * c[9] > c[1] for c in G.RAGGED_CONV_CASES for l in c[10])
    # the tile choice itself: 64-row tiles below two CTAs per SM, 64-column tiles when 128 would leave SMs idle
    assert G.simt_plan(16, 1000, 256, 1024, 9) == (128, 128) and G.simt_plan(2, 131, 1024, 256, 1) == (64, 64)
    h = _lib.lib()
    a = _lib.Conv1dArgs(x=16, w=16, y=16, B=1, T=128, Cin=24, N=16, taps=1)
    out = _lib.ConvSimtPlan()
    assert h.fs2_conv_simt_plan(ctypes.byref(a), 132, ctypes.byref(out)) == -2
    a.Cin, a.T = 16, 0
    assert h.fs2_conv_simt_plan(ctypes.byref(a), 132, ctypes.byref(out)) == -1


def test_fused_resblock_plan_respects_the_hardware_limits():
    """fs2_resstack_plan (pure host logic) over the shipped generator's kernel / dilation sets, every single-pair shape and a sweep of
    lengths: the halo covers the receptive radius, the output boxes tile the work item exactly in whole swizzle atoms, and shared memory
    and the consumer threads' accumulator + residual registers stay inside the SM's budget."""
    plan = _rs_plan
    cases = [(C, N, (3, 7, 11), ((1, 3, 5),) * 3) for C in (32, 64) for N in (1, 50, 392, 1000, 129536, 259072)]
    cases += [(C, N, (k,), ((d,),)) for C in (32, 64) for N in (40, 1000, 259072) for k in (3, 5, 7, 11) for d in (1, 3, 5)]
    cases += [(C, 5000, (3,), ((1, 3, 5),)) for C in (32, 64)] + [(64, 50, (3, 5), ((1, 2), (2, 6)))]
    for C, N, ks, dils in cases:
        rc, p = plan(C, N, ks, dils)
        assert rc == 0, (C, N, ks, dils, rc)
        radius = max(sum((k - 1) * d // 2 + (k - 1) // 2 for d in dd) for k, dd in zip(ks, dils))
        assert p["H"] >= radius and p["H"] % 4 == 0
        assert p["OBOX"] % 8 == 0 and 8 <= p["OBOX"] <= 256 and p["n_oboxes"] * p["OBOX"] == p["TILE"] and p["n_oboxes"] <= 12
        assert p["TILE"] == p["MT"] * 128 - 2 * p["H"]
        assert p["smem"] <= 227 * 1024 and p["acc_regs"] == p["MT"] * C <= 128
        assert 2 <= p["SB"] <= 8 and p["TPS"] * 64 * C == 8192
        assert p["n_items"] == 16 * -(-N // p["TILE"]) and p["grid"] == min(p["n_items"], 132)
    # refused: other widths, even kernels, taps reaching more than 32 rows outside a tile, table overflow
    assert plan(128, 1000, (3,), ((1,),))[0] == -2 and plan(32, 1000, (4,), ((1,),))[0] == -2
    assert plan(32, 1000, (11,), ((7,),))[0] == -2 and plan(32, 0, (3,), ((1,),))[0] == -1


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "fastspeech2_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f


def test_cpu_tensors_fail_loudly(lj_configs):
    import torch
    from fastspeech2_b200 import synth
    from fastspeech2_b200.model import FastSpeech2
    pc, mc = lj_configs
    m = FastSpeech2(pc, mc).eval()
    spk, texts, lens, L = synth.make_batch(1, 8)
    with pytest.raises(_lib.Fs2Error):
        m(spk, texts, lens, L)
