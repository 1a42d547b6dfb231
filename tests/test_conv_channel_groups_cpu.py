"""CPU: the tensor-core conv planner's channel-block groups (fs2_conv_tc_plan_t::NG).

A work item computes NG blocks of NB output channels from one resident input slab, so the slab ring must hold all C_in / 16 K-blocks
of the item (SA >= C_in / 16 <= 8) next to the weight ring and the staged epilogue tiles.  NG > 1 is planned only where that fits,
where at least four waves of items remain, and for one K-segment."""
import ctypes

from fastspeech2_b200 import _lib

BUDGET = 226 * 1024
B, FRAMES = 16, 1012                                   # the bench step: configs[2]


def _plan(B, T, Cin, N, taps, dil=1, res=False, accumulate=False, tc_variant=_lib.TC_VARIANT_F8, x_lens=0, num_sms=132):
    a = _lib.Conv1dArgs(x=0x1000, x_batch_stride=T * Cin, x_row_stride=Cin, B=B, T=T, Cin=Cin, w=0x1000, N=N, taps=taps, dilation=dil,
                        pad_left=(taps - 1) * dil // 2, w_tc=0x1000, y=0x1000, y_batch_stride=T * N, y_row_stride=N, alpha=1.0,
                        res=0x2000 if res else 0, res_batch_stride=T * N if res else 0, res_row_stride=N if res else 0,
                        accumulate=int(accumulate), tc_variant=tc_variant, x_lens=x_lens, lens_scale=1)
    out = _lib.ConvTcPlan()
    rc = _lib.lib().fs2_conv_tc_plan(ctypes.byref(a), num_sms, ctypes.byref(out))
    assert rc == 0, (B, T, Cin, N, taps, dil, rc)
    return _lib.fields(out)


def _check(p, Cin, N, T, Bn=B):
    assert p["smem"] <= BUDGET and 2 <= p["SB"] <= 8 and 1 <= p["SA"] <= 8
    assert p["n_items"] == (N // p["NB"]) * Bn * -(-T // 128)
    assert (N // p["NB"]) % p["NG"] == 0
    if p["NG"] > 1:
        assert p["SA"] >= Cin // 16 and p["n_items"] // p["NG"] >= 4 * 132 and p["grid"] == 132


def test_the_128_channel_resblock_convs_compute_both_blocks_from_one_slab():
    T = FRAMES * 64
    for k in (3, 7, 11):
        for d in (1, 3, 5):
            for res, acc in ((False, False), (True, False), (True, True)):
                p = _plan(B, T, 128, 128, k, d, res, acc)
                _check(p, 128, 128, T)
                assert p["NB"] == 64 and p["NG"] == 2 and p["SA"] == 8, (k, d, res, acc, p)


def test_slabs_that_do_not_fit_the_ring_keep_one_block_per_item():
    # C_in = 256 (stage 0's ResBlocks, stage 1's ConvTranspose groups) and 512 (stage 0's) need 16 and 32 slab stages
    for Cin, N, T, k in ((256, 256, FRAMES * 8, 3), (256, 256, FRAMES * 8, 11), (256, 512, FRAMES * 8, 2), (512, 1024, FRAMES, 2)):
        p = _plan(B, T, Cin, N, k)
        _check(p, Cin, N, T)
        assert p["NG"] == 1, (Cin, N, p)


def test_few_tiles_keep_the_parallelism():
    # 2 blocks x 4 x 66 tiles: 264 grouped items would be two waves on 132 SMs
    p = _plan(4, 66 * 128, 128, 128, 3)
    _check(p, 128, 128, 66 * 128, 4)
    assert p["NG"] == 1 and p["grid"] == 132
    p = _plan(4, 132 * 128, 128, 128, 3)
    _check(p, 128, 128, 132 * 128, 4)
    assert p["NG"] == 2


def test_segmented_convs_keep_one_block_per_item_and_ragged_ones_plan_as_padded():
    seg = _plan(16, 1024, 1024, 256, 1, tc_variant=_lib.TC_VARIANT_NB64 | _lib.TC_VARIANT_SEGMENTED)
    assert seg["NG"] == 1
    ragged = _plan(B, FRAMES * 64, 128, 128, 3, x_lens=0x3000)   # the plan of the padded shape: lengths stay on the device
    assert ragged == _plan(B, FRAMES * 64, 128, 128, 3) and ragged["NG"] == 2


def test_a_plan_without_groups_is_unchanged():
    # the split-fp16 layout at 128 output channels has one block: the NG = 1 plan (test_abi pins its ring depths)
    p = _plan(B, FRAMES * 64, 128, 128, 3, tc_variant=0)
    assert p["NB"] == 128 and p["NG"] == 1 and p["SA"] == 5
