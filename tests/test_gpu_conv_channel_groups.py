"""GPU: channel-block groups (fs2_conv_tc_plan_t::NG) change which CTA computes a block, never the bits.

A conv planned at NG = 2 must equal, bit for bit, the same conv computed one 64-channel block at a time (N = 64 per launch: one block,
so NG = 1), each block's launch reading its tiles from the same packed buffer, in the padded layout with every epilogue mode.  Plans
are made with the device's own SM count.  The windowed entry points are checked through Generator: stream() in one
window whose 128-channel stage is planned at NG = 2 against short windows planned at NG = 1, and a multi-generator pool large enough
for NG = 2 against each stream's own forward."""
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, ops, packing, synth
from tests.test_conv_channel_groups_cpu import _plan as _plan_at
from tests.test_gpu_conv_groups import block_tiles, device_sms
from tests.test_gpu_stream_multi import _run
from tests.test_gpu_stream_vocoder import _generator, _streamed

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _plan(*a, **k):
    return _plan_at(*a, num_sms=device_sms(), **k)


def _conv(x, w, b, dil, res, y, alpha, acc, out_act, w_tc):
    ops.conv1d(x, w, b, dilation=dil, pad_left=(w.shape[0] - 1) * dil // 2, in_act=L.ACT_LRELU, in_slope=0.1, out_act=out_act,
               out_slope=0.1, res=res, alpha=alpha, out=y, accumulate=acc, w_tc=w_tc, backend=L.CONV_TC, tc_variant=L.TC_VARIANT_F8)


@pytest.mark.parametrize("k,dil", [(3, 1), (11, 5)])
@pytest.mark.parametrize("mode", ["plain", "res", "res+acc"])
def test_grouped_blocks_equal_one_block_per_launch(k, dil, mode):
    Bn, T, C = 4, 132 * 128 + 37, 128                  # a partial last tile
    assert _plan(Bn, T, C, C, k, dil, mode != "plain", mode == "res+acc")["NG"] == 2
    assert _plan(Bn, T, C, 64, k, dil, mode != "plain", mode == "res+acc")["NG"] == 1
    g = torch.Generator().manual_seed(k * 10 + dil)
    x = torch.randn(Bn, T, C, generator=g).to(DEV)
    w = (torch.randn(k, C, C, generator=g) * (k * C) ** -0.5).to(DEV)
    b = (torch.randn(C, generator=g) * 0.1).to(DEV)
    res = torch.randn(Bn, T, C, generator=g).to(DEV) if mode != "plain" else None
    y0 = torch.randn(Bn, T, C, generator=g).to(DEV)
    acc, alpha, out_act = mode == "res+acc", (1 / 3 if mode == "res+acc" else 1.0), (L.ACT_LRELU if mode == "plain" else L.ACT_NONE)
    grouped, split = y0.clone(), y0.clone()
    w_tc = packing.pack_conv_tc(w.cpu(), f8=True).to(DEV)
    _conv(x, w, b, dil, res, grouped, alpha, acc, out_act, w_tc)
    for n in (0, 64):
        _conv(x, w[:, :, n:n + 64].contiguous(), b[n:n + 64], dil, None if res is None else res[:, :, n:n + 64], split[:, :, n:n + 64],
              alpha, acc, out_act, block_tiles(w_tc, n // 64, k, C, 64))
    torch.cuda.synchronize()
    assert torch.equal(grouped, split)


@pytest.mark.parametrize("ragged", [False, True])
def test_windowed_vocoder_with_groups_equals_short_windows(ragged):
    """One window over the whole batch (conv_tc_streams_kernel, the 128-channel stage planned at NG = 2) against 64-frame windows
    (NG = 1) and the offline forward."""
    gen = _generator(configs.HIFIGAN_CONFIG)
    Bn, frames = 4, 1100                               # 128-channel stage: 4 x 550 tiles x 2 blocks
    assert _plan(Bn, frames * 64, 128, 128, 3)["NG"] == 2 and _plan(Bn, 70 * 64, 128, 128, 3)["NG"] == 1
    mel = synth.make_mel(Bn, frames, seed=31).to(DEV)
    lens = torch.tensor([frames, 700, 1, frames - 3]) if ragged else None
    whole = _streamed(gen, mel, lens, frames)
    short = _streamed(gen, mel, lens, 64)
    torch.cuda.synchronize()
    assert torch.equal(whole, short) and torch.equal(whole, gen(mel, lens))


def test_multi_generator_pool_with_groups_equals_each_forward():
    """64 streams of two generators in one pool (windowed conv_tc_table_kernel, NG = 2 from the first tick's window on) against each
    stream's own generator's forward on that stream alone (one utterance: NG = 1)."""
    gens = [_generator(configs.HIFIGAN_CONFIG, seed=s) for s in (3, 11)]
    n, frames, chunk = 64, 80, 32
    assert _plan(n, chunk * 64, 128, 128, 3)["NG"] == 2 and _plan(1, frames * 64, 128, 128, 3)["NG"] == 1
    pool = gens[0].stream_pool(chunk_frames=chunk, generators=gens[1:])
    mels = [synth.make_mel(1, frames - k % 7, seed=60 + k)[0].to(DEV) for k in range(n)]
    which = [k % 2 for k in range(n)]
    out = _run(pool, mels, which, [0] * n)
    for k, mel in enumerate(mels):
        assert torch.equal(out[k], gens[which[k]](mel[None])), k
