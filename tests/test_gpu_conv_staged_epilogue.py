"""GPU: the edge cases of the conv kernel's staged epilogue inputs (residual / old y bulk-copied to shared memory per work item; the
K-segmented slice sum kept there), against tests/emul_cabi.py's contract with the per-element bars of test_gpu_tc_precision.py."""
import pytest
import torch

from fastspeech2_b200 import _lib as L, ops, packing
from tests import emul_cabi as E

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _case(B, T, Cin, N, k, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, Cin, generator=g)
    w = torch.randn(k, Cin, N, generator=g) * (k * Cin) ** -0.5
    return g, x, w, torch.randn(N, generator=g) * 0.1, torch.randn(B, T, N, generator=g), torch.randn(B, T, N, generator=g)


def _strided(t, pad, fill=0.0):
    """t as a [B, T, N] view of a wider buffer: row stride N + 2 * pad, first column at pad (16-byte aligned)"""
    B, T, N = t.shape
    big = torch.full((B, T, N + 2 * pad), fill, device=DEV)
    v = big[:, :, pad:pad + N]
    v.copy_(t.to(DEV))
    return big, v


def _run(x, w, bias, fmt, dil, res, y, alpha, accumulate, row_lens=None, x_lens=None, seg=False, in_act=L.ACT_LRELU, out_act=L.ACT_NONE):
    wt = packing.pack_conv_tc_segments(w) if seg else packing.pack_conv_tc(w, f8=fmt == "f8")
    variant = L.TC_VARIANT_NB64 | L.TC_VARIANT_SEGMENTED if seg else int(fmt == "f8")
    ops.conv1d(x.to(DEV), w.to(DEV), bias.to(DEV), dilation=dil, pad_left=(w.shape[0] - 1) * dil // 2, in_act=in_act, in_slope=0.1,
               out_act=out_act, out_slope=0.1, res=res, alpha=alpha, out=y, accumulate=accumulate, row_lens=row_lens, w_tc=wt.to(DEV),
               backend=L.CONV_TC, tc_variant=variant, x_lens=x_lens)
    torch.cuda.synchronize()


def _check(got, x, w, bias, fmt, dil, res, y0, alpha, row_lens=None, seg=False, in_act=L.ACT_LRELU, out_act=L.ACT_NONE):
    y_c, y64, S, R = E.tc_contract(x, w, bias, fmt, dil, (w.shape[0] - 1) * dil // 2, in_act, 0.1, out_act, 0.1, res, alpha, y0, row_lens,
                                   seg_cin=packing.SEG_CIN if seg else None)
    ea, eb = E.tc_errors(got.cpu(), y_c, y64, S, R)
    bar = E.TC_SEG_ACC_C if seg else E.TC_ACC_C
    assert ea <= bar and eb <= bar, (ea, eb, bar)


@pytest.mark.parametrize("fmt,N", [("split3", 128), ("f8", 64), ("split3", 48)])
def test_partial_tile_residual_and_accumulate(fmt, N):
    """T not a multiple of 128: the last tile's staged rows stop at T"""
    _, x, w, b, r, y0 = _case(2, 300, 64, N, 3, 1)
    y = y0.to(DEV).clone()
    _run(x, w, b, fmt, 3, r.to(DEV), y, 0.5, True)
    _check(y, x, w, b, fmt, 3, r, y0, 0.5)


@pytest.mark.parametrize("fmt", ["split3", "f8"])
def test_strided_residual_and_y(fmt):
    """residual and y as views with row stride != N, accumulate"""
    N = 64
    _, x, w, b, r, y0 = _case(3, 257, 32, N, 5, 2)
    rbig, rv = _strided(r, 8)
    ybig, yv = _strided(y0, 12, fill=7.0)
    _run(x, w, b, fmt, 1, rv, yv, 1 / 3, True)
    _check(yv, x, w, b, fmt, 1, r, y0, 1 / 3)
    assert torch.all(ybig[:, :, :12] == 7.0) and torch.all(ybig[:, :, 12 + N:] == 7.0)     # the pad columns stay untouched


@pytest.mark.parametrize("fmt,N", [("split3", 256), ("f8", 256)])
def test_several_items_per_cta_and_channel_blocks(fmt, N):
    """>= 2 work items per CTA of a 132-SM grid over 2 (split3) or 4 (f8) channel blocks, residual + accumulate"""
    _, x, w, b, r, y0 = _case(4, 128 * 40 - 5, 32, N, 3, 3)
    y = y0.to(DEV).clone()
    _run(x, w, b, fmt, 1, r.to(DEV), y, 0.5, True)
    _check(y, x, w, b, fmt, 1, r, y0, 0.5)


@pytest.mark.parametrize("fmt", ["split3", "f8"])
def test_ragged_accumulate_leaves_rows_past_the_utterance_alone(fmt):
    """ragged x_lens with row_lens: rows < n_b against a B = 1 run of that utterance; rows >= n_b of y hold NaN and must keep it"""
    B, T, N = 3, 400, 64
    _, x, w, b, r, y0 = _case(B, T, 64, N, 3, 4)
    n = [400, 1, 129]
    row_lens = torch.tensor([300, 1, 100], dtype=torch.int32)
    for i, nb in enumerate(n):
        y0[i, nb:] = float("nan")
    y = y0.to(DEV).clone()
    _run(x, w, b, fmt, 5, r.to(DEV), y, 0.5, True, row_lens=row_lens.to(DEV), x_lens=torch.tensor(n, dtype=torch.int32, device=DEV))
    for i, nb in enumerate(n):
        assert torch.isnan(y[i, nb:]).all(), i
        _check(y[i:i + 1, :nb], x[i:i + 1, :nb], w, b, fmt, 5, r[i:i + 1, :nb], y0[i:i + 1, :nb], 0.5, row_lens=row_lens[i:i + 1])


@pytest.mark.parametrize("accumulate", [False, True])
def test_segmented_with_residual(accumulate):
    """K-segmented conv (slice sum kept in shared memory) with a residual, several items per CTA, a partial last tile"""
    _, x, w, b, r, y0 = _case(8, 128 * 33 + 17, 512, 128, 3, 5)
    y = y0.to(DEV).clone()
    _run(x, w, b, "split3", 1, r.to(DEV), y, 1.0, accumulate, seg=True, in_act=L.ACT_NONE)
    _check(y, x, w, b, "split3", 1, r, y0 if accumulate else None, 1.0, seg=True, in_act=L.ACT_NONE)
