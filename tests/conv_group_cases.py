"""Channel-block group cases for the tensor-core conv (TEST INFRASTRUCTURE, shared by tests/test_conv_groups_cpu.py and
tests/test_gpu_conv_groups.py).

A work item of the tensor-core conv is one 128-row tile x NG channel blocks of NB output channels: the item's C_in / 16 slab stages
are loaded once and read NG times, the consumers rewind their slab cursor between passes and release the stages on the last one
(Ring::rewind, ring_release_last), and the weight producer decodes every (item, block) unit into a 16-slot ring (TcSlot).  The planner
(conv_tc_plan) picks NG > 1 from the shape and the SM count, so every case here names its layer and a target NG, and choose_batch
finds the batch at which the planner picks exactly that NG on a given number of SMs.  Each case carries the classes it covers
(`cls`): format and block width, NG with a group index above 0, where the item's slab falls in the 8-stage slab ring, taps per
weight stage, epilogue, row bounds, strides, the slot ring's wrap, and the shipped layers that reach NG > 1 at the benchmark's
shapes.
"""
import ctypes

from fastspeech2_b200 import _lib

FMT_VARIANT = {"split3": 0, "f8": _lib.TC_VARIANT_F8}
SA_MAX = 8                                             # conv_tc_kernel.cuh: TC_SA_MAX, the slab ring's stages
SLOTS = 16                                             # TC_SLOTS: the unit slot ring


def nb_of(fmt, N):
    """The block width the planner gives a plain (not NB64) tile format: conv_tc_nb(N, 64 for f8, 128 for split3)."""
    nb_max = 64 if fmt == "f8" else 128
    if N <= nb_max:
        return N
    return next(nb for nb in range(nb_max, 15, -16) if N % nb == 0)


def case(name, cls, fmt, Cin, N, taps, NG, dil=1, pad=None, T=300, in_act=_lib.ACT_NONE, out_act=_lib.ACT_NONE, bias=True, res=False,
         acc=False, alpha=1.0, lens=None, x_cols=None, y_cols=None, x=("scale", 0)):
    """One layer: fmt, Cin -> N, taps at dilation dil (pad_left: centred by default); T rows per utterance (T % 128 != 0: every CTA
    has partial tiles); NG the group size the planner must pick.  lens: None, "row_lens" (rows at or past the length are zeroed) or
    "x_lens" (a ragged batch with 0- and 1-row utterances).  x_cols = (total, offset): x is a column slice of a wider row, whose
    batch stride also skips 5 extra rows; y_cols = (total, offset): y is a column slice of rows of `total` floats (a ConvTranspose
    phase group writes (u / 2) C_out of u C_out).  x: the activation spec of tests/tc_cases.make_x."""
    if pad is None:
        pad = (taps - 1) * dil // 2
    return dict(name=name, cls=tuple(cls), fmt=fmt, Cin=Cin, N=N, taps=taps, NG=NG, dil=dil, pad=pad, T=T, in_act=in_act,
                out_act=out_act, bias=bias, res=res, acc=acc, alpha=alpha, lens=lens, x_cols=x_cols, y_cols=y_cols, x=x)


L_, TANH, RELU = _lib.ACT_LRELU, _lib.ACT_TANH, _lib.ACT_RELU

CASES = [
    # ---- format and block width: f8 (TG = 2) at NB 16 / 32 / 48 / 64, split3 (TG = 1) at NB 80 / 96 / 112 / 128 and NB = 16
    case("f8_nb16_25blk", ["f8", "nb16", "ng5"], "f8", 64, 400, 3, 5),
    case("f8_nb32_5blk", ["f8", "nb32"], "f8", 32, 160, 3, 5, out_act=RELU),
    case("f8_nb48_3blk", ["f8", "nb48", "ng3"], "f8", 128, 144, 3, 3, in_act=L_),
    case("f8_nb48_6blk_ng3", ["f8", "nb48", "ng3", "group>0"], "f8", 80, 288, 5, 3, out_act=L_),
    case("f8_nb48_6blk_ng2", ["f8", "nb48", "ng2", "group>0", "no_bias"], "f8", 16, 288, 1, 2, bias=False),
    case("f8_nb64_4blk_ng2", ["f8", "nb64", "ng2", "group>0", "kb4", "slab_next_resident"], "f8", 64, 256, 3, 2, in_act=L_),
    case("f8_nb64_8blk_ng4", ["f8", "nb64", "ng4", "group>0", "kb2", "slab_next_resident"], "f8", 32, 512, 2, 4),
    case("f8_nb64_16blk_ng8", ["f8", "nb64", "ng8", "group>0", "kb8", "slots>16"], "f8", 128, 1024, 3, 8, in_act=L_, out_act=L_),
    case("f8_nb64_16blk_ng4", ["f8", "nb64", "ng4", "group>0", "kb7", "slab_wraps"], "f8", 112, 1024, 1, 4),
    case("split3_nb80_2blk", ["split3", "nb80", "ng2"], "split3", 80, 160, 3, 2),
    case("split3_nb80_4blk_ng2", ["split3", "nb80", "ng2", "group>0", "kb5", "slab_wraps"], "split3", 80, 320, 5, 2, out_act=TANH),
    case("split3_nb80_3blk_ng3", ["split3", "nb80", "ng3"], "split3", 32, 240, 7, 3, out_act=RELU),
    case("split3_nb96_6blk_ng3", ["split3", "nb96", "ng3", "group>0", "kb4"], "split3", 64, 576, 3, 3),
    case("split3_nb96_6blk_ng2", ["split3", "nb96", "ng2", "group>0", "kb1", "slab_next_resident"], "split3", 16, 576, 11, 2, dil=3),
    case("split3_nb112_4blk_ng2", ["split3", "nb112", "ng2", "group>0", "kb7", "slab_wraps"], "split3", 112, 448, 2, 2, in_act=L_),
    case("split3_nb112_4blk_ng4", ["split3", "nb112", "ng4"], "split3", 32, 448, 3, 4, out_act=L_),
    case("split3_nb128_8blk_ng4", ["split3", "nb128", "ng4", "group>0", "kb2"], "split3", 32, 1024, 1, 4, bias=False),
    case("split3_nb128_8blk_ng2", ["split3", "nb128", "ng2", "group>0", "kb8"], "split3", 128, 1024, 3, 2),
    case("split3_nb128_16blk_ng8", ["split3", "nb128", "ng8", "group>0", "kb1", "slots>16"], "split3", 16, 2048, 2, 8, in_act=L_),
    case("split3_nb16_11blk", ["split3", "nb16", "ng11", "slots>16"], "split3", 64, 176, 3, 11),
    case("f8_nb64_12blk_ng3", ["f8", "nb64", "ng3", "group>0", "kb5", "slab_wraps"], "f8", 80, 768, 7, 3, out_act=TANH),
    # ---- taps per weight stage (TPS 4 from 5 taps on) and dilation up to the 256-row halo
    case("taps5_4+1", ["taps5"], "f8", 64, 256, 5, 2, dil=2),
    case("taps7_4+3", ["taps7"], "split3", 64, 256, 7, 2, dil=4),
    case("taps11_4+4+3", ["taps11"], "f8", 32, 512, 11, 4, dil=5, in_act=L_),
    case("taps2_dil256", ["taps2", "halo256"], "f8", 32, 256, 2, 2, dil=256, pad=128),
    case("taps3_dil128", ["taps3", "halo256"], "split3", 16, 256, 3, 2, dil=128),
    # ---- the slab ring: SA == K-blocks < 8, SA between K-blocks and 8, and a 2-stage weight ring (the wide halos)
    case("wide_halo_sa_eq_kb", ["sa==kb<8", "kb4", "taps11"], "split3", 64, 256, 11, 2, dil=25),
    case("wide_halo_sb2", ["sb2", "kb6", "taps11"], "split3", 96, 512, 11, 4, dil=25),
    case("wide_halo_kb<sa<8", ["kb<sa<8", "kb4", "taps11"], "f8", 64, 256, 11, 4, dil=25, out_act=L_),
    # ---- epilogues: residual, residual + accumulate + alpha, with and without bias
    case("res_f8", ["res"], "f8", 128, 256, 3, 2, in_act=L_, res=True),
    case("res_acc_f8", ["res+acc"], "f8", 64, 512, 7, 4, dil=3, in_act=L_, res=True, acc=True, alpha=1 / 3),
    case("res_acc_split3_nb80", ["res+acc", "nb80", "no_bias"], "split3", 32, 320, 3, 2, res=True, acc=True, alpha=0.5, bias=False),
    case("res_split3_nb128", ["res", "nb128"], "split3", 16, 512, 5, 2, res=True, out_act=RELU),
    case("res_acc_f8_nb32", ["res+acc", "nb32", "kb1"], "f8", 16, 160, 3, 5, res=True, acc=True, alpha=0.25),
    # ---- row bounds: row_lens masking, ragged x_lens with 0- and 1-row utterances
    case("row_lens_f8", ["row_lens"], "f8", 64, 512, 3, 4, lens="row_lens", out_act=L_),
    case("row_lens_split3_res", ["row_lens", "res"], "split3", 80, 320, 5, 2, lens="row_lens", res=True),
    case("x_lens_f8", ["x_lens"], "f8", 128, 256, 3, 2, lens="x_lens", in_act=L_),
    case("x_lens_split3_acc", ["x_lens", "res+acc"], "split3", 32, 448, 7, 2, lens="x_lens", res=True, acc=True, alpha=1 / 3),
    case("x_lens_f8_ng8", ["x_lens", "ng8", "slots>16"], "f8", 16, 1024, 2, 8, lens="x_lens"),
    # ---- strides: a column slice of x, a column slice of y, both
    case("x_strided", ["x_strided"], "f8", 64, 512, 3, 4, x_cols=(96, 16)),
    case("y_strided", ["y_strided"], "split3", 32, 448, 3, 2, y_cols=(512, 32)),
    case("xy_strided_res", ["x_strided", "y_strided", "res"], "f8", 80, 256, 5, 2, x_cols=(128, 40), y_cols=(320, 64), res=True),
    # ---- operand magnitudes away from N(0, 1)
    case("x2^-12_f8", ["x2^-12"], "f8", 64, 256, 3, 4, x=("scale", -12)),
    case("chan_split3", ["x_chan"], "split3", 32, 512, 3, 4, x=("chan", -14, 4)),
    # ---- the shipped layers that plan NG > 1 at the benchmark's shapes, verbatim
    case("postnet_conv0_ng2", ["shipped", "postnet0", "tanh"], "f8", 80, 512, 5, 2, out_act=TANH, T=1012),
    case("postnet_conv0_ng4", ["shipped", "postnet0", "tanh", "taps5", "kb5", "slab_wraps"], "f8", 80, 512, 5, 4, out_act=TANH,
         T=1012),
    case("postnet_conv0_ng8", ["shipped", "postnet0", "tanh", "ng8", "slots>16"], "f8", 80, 512, 5, 8, out_act=TANH, T=2006),
    case("v1_conv_pre_ng2", ["shipped", "v1_conv_pre", "taps7", "kb5", "slab_wraps"], "split3", 80, 512, 7, 2, T=1012),
    case("v1_conv_pre_ng4", ["shipped", "v1_conv_pre", "ng4"], "split3", 80, 512, 7, 4, T=2006),
    case("v2_ups0_phase_a_ng2", ["shipped", "v2_ups0", "phase_group", "taps2", "kb8"], "f8", 128, 256, 2, 2, pad=1, in_act=L_,
         y_cols=(512, 0), T=1012),
    case("v2_ups0_phase_b_ng4", ["shipped", "v2_ups0", "phase_group", "ng4"], "f8", 128, 256, 2, 4, pad=0, in_act=L_,
         y_cols=(512, 256), T=2006),
    case("v2_ups1_phase_b_ng2", ["shipped", "v2_ups1", "phase_group", "kb4"], "f8", 64, 128, 2, 2, pad=0, in_act=L_,
         y_cols=(256, 128), T=1012),
    case("v1_c128_conv1_k3", ["shipped", "v1_c128", "taps3"], "f8", 128, 128, 3, 2, dil=3, in_act=L_, out_act=L_),
    case("v1_c128_conv1_k11", ["shipped", "v1_c128", "taps11"], "f8", 128, 128, 11, 2, dil=5, in_act=L_),
    case("v1_c128_conv2_k7_res_acc", ["shipped", "v1_c128", "res+acc"], "f8", 128, 128, 7, 2, in_act=L_, res=True, acc=True,
         alpha=1 / 3),
]

# Every class section 1 of the test plan names: each must be covered by at least one case (checked on the CPU).
REQUIRED_CLASSES = {"f8", "split3", "nb16", "nb32", "nb48", "nb64", "nb80", "nb96", "nb112", "nb128", "ng2", "ng3", "ng4", "ng8",
                    "group>0", "kb1", "kb2", "kb4", "kb5", "kb7", "kb8", "slab_wraps", "slab_next_resident", "sa==kb<8", "kb<sa<8",
                    "sb2", "taps2", "taps3", "taps5", "taps7", "taps11", "halo256", "tanh", "res", "res+acc", "no_bias", "row_lens",
                    "x_lens", "x_strided", "y_strided", "phase_group", "slots>16", "shipped"}


def classes(c):
    """The case's labels plus the classes derived from its shape (so that a label cannot claim what the shape does not do)."""
    out = set(c["cls"])
    out.add(c["fmt"])
    out.add(f"ng{c['NG']}")
    out.add(f"kb{c['Cin'] // 16}")
    out.add(f"taps{c['taps']}")
    out.add(f"nb{nb_of(c['fmt'], c['N'])}")
    if c["out_act"] == TANH:
        out.add("tanh")
    return out


def conv_args(c, B, x_ptr=0x1000, lens_ptr=0):
    """fs2_conv1d_args of case c at batch B (pointer values only for the planner's alignment checks)."""
    T, Cin, N = c["T"], c["Cin"], c["N"]
    xt = c["x_cols"][0] if c["x_cols"] else Cin
    yt = c["y_cols"][0] if c["y_cols"] else N
    xbs = (T + 5) * xt if c["x_cols"] else T * Cin
    return _lib.Conv1dArgs(x=x_ptr, x_batch_stride=xbs, x_row_stride=xt, B=B, T=T, Cin=Cin, w=0x1000, N=N, taps=c["taps"],
                           dilation=c["dil"], pad_left=c["pad"], w_tc=0x1000, y=0x1000, y_batch_stride=T * yt, y_row_stride=yt,
                           alpha=c["alpha"], in_act=c["in_act"], in_slope=0.1, out_act=c["out_act"], out_slope=0.1,
                           res=0x2000 if c["res"] else 0, res_batch_stride=T * N if c["res"] else 0,
                           res_row_stride=N if c["res"] else 0, accumulate=int(c["acc"]), tc_variant=FMT_VARIANT[c["fmt"]],
                           x_lens=0x3000 if c["lens"] == "x_lens" else 0, lens_scale=1,
                           row_lens=0x3000 if c["lens"] == "row_lens" else 0)


def plan_args(a, num_sms):
    """fs2_conv_tc_plan of fs2_conv1d_args a on num_sms SMs, as a dict."""
    out = _lib.ConvTcPlan()
    rc = _lib.lib().fs2_conv_tc_plan(ctypes.byref(a), num_sms, ctypes.byref(out))
    assert rc == 0, rc
    return _lib.fields(out)


def plan(c, B, num_sms):
    return plan_args(conv_args(c, B), num_sms)


def choose_batch(c, num_sms):
    """The smallest batch at which the planner picks c's NG on num_sms SMs, moved up until the grid does not divide the items, so that
    some CTAs run one item fewer than others.  The planner takes the largest divisor NG of the block count with at least 4 waves of
    items, n_items / NG >= 4 num_sms, so below this batch it picks a smaller NG and far above it a larger one."""
    nblk = c["N"] // nb_of(c["fmt"], c["N"])
    tiles = -(-c["T"] // 128)
    B = -(-4 * num_sms * c["NG"] // (nblk * tiles))
    for _ in range(8):
        p = plan(c, B, num_sms)
        if p["NG"] == c["NG"] and (p["n_items"] // p["NG"]) % p["grid"]:
            return B
        B += 1
    raise AssertionError(f"{c['name']}: no batch near {B} plans NG = {c['NG']} on {num_sms} SMs (last plan {p})")


def lens_of(c, B):
    """The per-utterance lengths of a case with lens: first and last utterances long (they carry the fp64 check), a 0-row and a
    1-row utterance, and the rest spread over [0, T]."""
    T = c["T"]
    lens = [(b * 7919 + 13) % (T + 1) for b in range(B)]
    lens[0], lens[-1] = T, T - 37
    if B > 3:
        lens[1], lens[2] = 0, 1
    return lens
