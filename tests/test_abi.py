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
             9: _lib.AcousticModel, 10: _lib.EncodeArgs, 11: _lib.DecodeArgs, 12: _lib.VocoderModel, 13: _lib.VocoderArgs, 14: _lib.ResstackArgs, 15: _lib.WavInt16Args}
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


def _plan(h, B, T, Cin, N, taps, dil=1, num_sms=132, x=0x1000, x_row_stride=None):
    a = _lib.Conv1dArgs(x=x, x_batch_stride=T * (x_row_stride or Cin), x_row_stride=x_row_stride or Cin, B=B, T=T, Cin=Cin, w=0x1000, N=N, taps=taps,
                        dilation=dil, pad_left=(taps - 1) * dil // 2, w_tc=0x1000, y=0x1000, y_batch_stride=T * N, y_row_stride=N, alpha=1.0)
    out = (ctypes.c_int32 * 12)()
    rc = h.fs2_conv_tc_plan(ctypes.byref(a), num_sms, out)
    keys = ("NB", "MT", "TG", "SA", "SB", "TPS", "R", "acc_regs", "tiles_per_batch", "n_items", "grid", "smem")
    return rc, dict(zip(keys, out))


def test_tensor_core_conv_launch_plan_respects_the_hardware_limits():
    """Host-side heuristics of the wgmma conv (work-item shape, ring depths, register / shared-memory budget) for every layer shape of
    both models at the BASELINE batch sizes, plus a sweep: no plan may exceed 227 KB of shared memory, 64 accumulator registers per
    consumer thread, the register-ring row capacity or the ring maxima, and the work items must cover the problem exactly."""
    h = _lib.lib()
    shapes = []
    for B, T in ((1, 7), (1, 1012), (16, 1012), (64, 2032)):
        shapes += [(B, T, 256, 768, 1, 1), (B, T, 256, 256, 1, 1), (B, T, 256, 1024, 9, 1), (B, T, 1024, 256, 1, 1), (B, T, 256, 80, 1, 1),
                   (B, T, 80, 512, 5, 1), (B, T, 512, 512, 5, 1), (B, T, 512, 80, 5, 1), (B, T, 128, 2048, 1, 1), (B, T, 2048, 128, 1, 1)]
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
        assert p["MT"] == 1 and p["TG"] == (2 if p["NB"] <= 64 else 1)
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
            out = (ctypes.c_int32 * 12)()
            assert h.fs2_conv_tc_plan(ctypes.byref(a), 132, out) == 0 and out[0] == h.fs2_conv_tc_block_f8(n) and out[2] == 2, n
    # ring depths per shape class: short kernels get the deepest slab ring, wide kernels share one weight stage between four taps
    assert _plan(h, 16, 64768, 128, 128, 3)[1]["SA"] == 5 and _plan(h, 16, 64768, 128, 128, 11, 5)[1]["TPS"] == 4
    # refused shapes: C_in % 16, N % 16, misaligned or oddly strided x, halo beyond the slab
    assert _plan(h, 1, 128, 24, 16, 1)[0] == -2 and _plan(h, 1, 128, 16, 24, 1)[0] == -2
    assert _plan(h, 1, 128, 16, 16, 1, x=0x1010)[0] == -2 and _plan(h, 1, 128, 16, 16, 1, x_row_stride=20)[0] == -2
    assert _plan(h, 1, 4096, 16, 16, 11, 30)[0] == -2


def test_fused_resblock_plan_respects_the_hardware_limits():
    """fs2_resstack_plan (pure host logic) over the shipped generator's kernel / dilation sets, every single-pair shape and a sweep of
    lengths: the halo covers the receptive radius, the output boxes tile the work item exactly in whole swizzle atoms, and shared memory
    and the consumer threads' accumulator + residual registers stay inside the SM's budget."""
    h = _lib.lib()

    def plan(C, N, ks, dils, B=16):
        a = _lib.ResstackArgs(B=B, N=N, C=C, n_kernels=len(ks), n_dil=len(dils[0]))
        for j, k in enumerate(ks):
            a.k[j] = k
            for d, dv in enumerate(dils[j]):
                a.dil[j][d] = dv
        out = (ctypes.c_int32 * 12)()
        rc = h.fs2_resstack_plan(ctypes.byref(a), 132, out)
        keys = ("MT", "H", "TILE", "items", "grid", "SB", "smem", "regs", "obox", "n_oboxes", "TPS", "indep")
        return rc, dict(zip(keys, out))

    cases = [(C, N, (3, 7, 11), ((1, 3, 5),) * 3) for C in (32, 64) for N in (1, 50, 392, 1000, 129536, 259072)]
    cases += [(C, N, (k,), ((d,),)) for C in (32, 64) for N in (40, 1000, 259072) for k in (3, 5, 7, 11) for d in (1, 3, 5)]
    cases += [(C, 5000, (3,), ((1, 3, 5),)) for C in (32, 64)] + [(64, 50, (3, 5), ((1, 2), (2, 6)))]
    for C, N, ks, dils in cases:
        rc, p = plan(C, N, ks, dils)
        assert rc == 0, (C, N, ks, dils, rc)
        radius = max(sum((k - 1) * d // 2 + (k - 1) // 2 for d in dd) for k, dd in zip(ks, dils))
        assert p["H"] >= radius and p["H"] % 4 == 0
        assert p["obox"] % 8 == 0 and 8 <= p["obox"] <= 256 and p["n_oboxes"] * p["obox"] == p["TILE"] and p["n_oboxes"] <= 12
        assert p["indep"] == 0 and p["TILE"] == p["MT"] * 128 - 2 * p["H"]
        assert p["smem"] <= 227 * 1024 and p["regs"] == p["MT"] * C <= 128
        assert 2 <= p["SB"] <= 8 and p["TPS"] * 64 * C == 8192
        assert p["items"] == 16 * -(-N // p["TILE"]) and p["grid"] == min(p["items"], 132)
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
