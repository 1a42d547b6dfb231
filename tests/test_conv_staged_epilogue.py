"""The conv kernel's staged epilogue inputs, checked without a GPU.

conv_tc_kernel reads the residual and the y it accumulates into from shared memory, where a staging warp bulk-copies them while the
work item's MMAs run.  A plain 64-bit global load of them in the epilogue would sit behind the previous y store (y may alias both),
one DRAM round trip per 8 columns with no MMA issuing.  The SASS must therefore hold no non-constant global load of 64 bits or wider
(bias, weights and activations go through the read-only path; the ragged lengths are 32-bit loads).  The launch plan budgets the
staging tiles exactly when a residual, accumulate or K-segments need them, within the 227 KB a block may use.
"""
import ctypes
import re

import pytest

from fastspeech2_b200 import _lib
from tests import test_sass_pipeline as S

TILE_ROWS, PAD, CWARPS = 128, 8, 8


def test_no_wide_non_constant_global_loads_in_the_conv_kernel(sass):
    found = 0
    for name, text in sass.items():
        if S._kernel(name) != "conv_tc_kernel":
            continue
        found += 1
        wide = re.findall(r"\bLDG\.E\.(?:64|128)\b(?!\.CONSTANT)[^;]*", text)
        assert not wide, f"{name}: {len(wide)} wide global loads outside the read-only path, e.g. {wide[0]}"
    assert found == S.N_INSTANTIATIONS["conv_tc_kernel"]


@pytest.fixture(scope="module")
def sass():
    """{mangled name: SASS text} of every tensor-core kernel"""
    funcs, name = {}, None
    for line in S._dump("-sass").splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if S._kernel(m.group(1)) else None
            if name:
                funcs[name] = []
        elif name:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


def _plan(B, T, Cin, N, taps, dil=1, res=False, accumulate=False, tc_variant=0):
    a = _lib.Conv1dArgs(x=0x1000, x_batch_stride=T * Cin, x_row_stride=Cin, B=B, T=T, Cin=Cin, w=0x1000, N=N, taps=taps, dilation=dil,
                        pad_left=(taps - 1) * dil // 2, w_tc=0x1000, y=0x1000, y_batch_stride=T * N, y_row_stride=N, alpha=1.0,
                        res=0x2000 if res else 0, res_batch_stride=T * N if res else 0, res_row_stride=N if res else 0,
                        accumulate=int(accumulate), tc_variant=tc_variant)
    out = _lib.ConvTcPlan()
    rc = _lib.lib().fs2_conv_tc_plan(ctypes.byref(a), 132, ctypes.byref(out))
    return rc, _lib.fields(out)


def _shapes():
    """every tensor-core conv shape of both models at the BASELINE batch sizes: (B, T, Cin, N, taps, dil, variant)"""
    out = []
    for B, T in ((1, 7), (16, 1012), (64, 2032)):
        for v in (0, _lib.TC_VARIANT_F8):
            out += [(B, T, 256, 768, 1, 1, v), (B, T, 256, 256, 1, 1, v), (B, T, 256, 1024, 9, 1, v), (B, T, 1024, 256, 1, 1, v),
                    (B, T, 80, 512, 5, 1, v), (B, T, 512, 512, 5, 1, v), (B, T, 512, 80, 5, 1, v)]
            t, c = T, 512
            for u in (8, 8, 2, 2):
                t, c = t * u, c // 2
                out += [(B, t, c, c, k, d, v) for k in (3, 7, 11) for d in (1, 3, 5)]
        seg = _lib.TC_VARIANT_NB64 | _lib.TC_VARIANT_SEGMENTED
        out += [(B, T, 256, 768, 1, 1, seg), (B, T, 256, 256, 1, 1, seg), (B, T, 256, 1024, 9, 1, seg), (B, T, 1024, 256, 1, 1, seg),
                (B, T, 256, 256, 3, 1, seg)]
    return out


def test_staging_is_budgeted_exactly_when_needed():
    for B, T, Cin, N, k, d, v in _shapes():
        nseg = k * (Cin // 256) if v & _lib.TC_VARIANT_SEGMENTED else 1
        rc, base = _plan(B, T, Cin, N, k, d, tc_variant=v)
        assert rc == 0, (B, T, Cin, N, k, d, v)
        for res, acc in ((False, False), (True, False), (False, True), (True, True)):
            rc, p = _plan(B, T, Cin, N, k, d, res=res, accumulate=acc, tc_variant=v)
            assert rc == 0, (B, T, Cin, N, k, d, v, res, acc)
            tiles = int(res) + int(acc or nseg > 1)
            staged = 2 * CWARPS * 8 + tiles * TILE_ROWS * (p["NB"] + PAD) * 4 if tiles else 0
            ring = p["smem"] - staged
            assert p["smem"] <= 227 * 1024, (B, T, Cin, N, k, d, v, res, acc, p)
            assert 2 <= p["SA"] <= 8 and 2 <= p["SB"] <= 8 and 1 <= p["TPS"] <= (1 if nseg > 1 else k)
            # what is not staging is exactly the rings the plan chose (slabs, weight stages, ring barriers)
            a_stage, b_stage = 2 * 2 * p["R"] * 16, p["TPS"] * 2 * 2 * p["NB"] * 16
            assert ring == p["SA"] * a_stage + p["SB"] * b_stage + (2 * 8 + 2 * 8) * 8 + 16, (B, T, Cin, N, k, d, v, res, acc, p)
            if tiles == 0:
                assert p == base                                  # unstaged shapes keep their plan
            for key in ("NB", "TG", "R", "tiles_per_batch", "n_items", "grid"):
                assert p[key] == base[key]
