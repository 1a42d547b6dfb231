"""GPU: V1's 128-channel stage with Generator.wide_pairs (its k = 3 pairs on fs2_resstack's 128-channel entry points, tiles packed at
NB = 128): the waveform against the fp64 CPU oracle at the 1e-4 bar and bit for bit against the default (per-layer) stage, ragged utterances as
if alone, and streamed chunks bit for bit equal to forward."""
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from oracle import fs2_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
H = AttrDict(configs.HIFIGAN_CONFIG)


def _gen(wide):
    g = Generator(H)
    g.load_state_dict(synth.hifigan_state_dict(H, seed=1))
    g = g.eval().to(DEV)
    g.wide_pairs = wide
    return g


def test_wide_pairs_vs_fp64_oracle_and_default():
    wide, base = _gen(True), _gen(False)
    assert wide.effective_masks()[2] >> 8 == 0b10                  # V1's 128-channel stage is stage 1
    mel = synth.make_mel(2, 40, seed=2)
    kw = dict(upsample_rates=H.upsample_rates, upsample_kernel_sizes=H.upsample_kernel_sizes,
              resblock_kernel_sizes=H.resblock_kernel_sizes, resblock_dilation_sizes=H.resblock_dilation_sizes, dtype=torch.float64)
    ref = O.hifigan_forward(synth.hifigan_state_dict(H, seed=1), mel.double(), **kw)
    launches = {}
    for name, g in (("wide", wide), ("base", base)):
        g(mel.to(DEV))                                              # packs the weights
        torch.cuda.synchronize()
        n0 = L.lib().fs2_kernel_launch_count()
        out = g(mel.to(DEV))
        launches[name] = (L.lib().fs2_kernel_launch_count() - n0, out)
    (nw, w), (nb, b) = launches["wide"], launches["base"]
    assert nw == nb - 3                                             # three pair launches in place of six per-layer convs
    assert torch.isfinite(w).all()
    assert (w.cpu().double() - ref).abs().max().item() < 1e-4
    # the pair kernel forms the same operand splits and sums each output row's products in the per-layer conv's order
    assert torch.equal(w, b)


def test_wide_pairs_ragged_and_streamed_bit_for_bit():
    g = _gen(True)
    mel = synth.make_mel(3, 70, seed=3).to(DEV)
    lens = torch.tensor([70, 41, 9], device=DEV)
    full = g(mel, mel_lens=lens)
    up = full.shape[-1] // 70
    for b, n in enumerate(lens.tolist()):
        alone = g(mel[b:b + 1, :, :n])
        assert torch.equal(full[b, :, :n * up], alone[0]), b
    for ml in (None, lens):
        ref = g(mel, mel_lens=ml)
        chunks = torch.cat([w for _, w in g.stream(mel, mel_lens=ml, chunk_frames=16)], dim=-1)
        assert torch.equal(chunks, ref)
    pool = g.stream_pool(chunk_frames=16)
    h = pool.add(mel[1, :, :41])
    got = []
    while len(pool):
        got += [w for hh, _, w in pool.step() if hh == h]
    assert torch.equal(torch.cat(got, dim=-1), g(mel[1:2, :, :41]))
