"""GPU: FastSpeech2 in ragged mode (fs2_acoustic_encode_ragged / fs2_acoustic_decode_ragged, FastSpeech2.forward(ragged=True)).

The contract (include/fs2b200.h): utterance b of a ragged call equals, bit for bit, the default-mode call on that utterance alone,
m(spk[b:b+1], texts[b:b+1, :n], src_lens[b:b+1], n, ...) with n = src_lens[b] (targets sliced the same way, max_mel_len = mel_lens[b]
when teacher-forced): mel_lens and durations equal, predictions equal on the utterance's own columns, mel / postnet_mel equal on its
own rows and exact zeros beyond them.  Every ragged call here runs on a model workspace filled with NaN first, so a single read of a
row outside an utterance would show up as NaN in its outputs."""
import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, ops, packing, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from fastspeech2_b200.model import FastSpeech2
from oracle import fs2_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
MEL_TOL = 1e-3
TC_MASKS = {"default": None, "fp32_cuda_cores": 0}


def _model(cfgs, seed, tc_mask=None, sd=None):
    pc, mc = cfgs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=seed) if sd is None else sd
    m = FastSpeech2(pc, mc)
    m.load_state_dict(sd)
    if tc_mask is not None:
        m.tc_mask = tc_mask
    return m.to(DEV).eval(), sd


def _dev(xs):
    return [x.to(DEV) if torch.is_tensor(x) else x for x in xs]


def _ragged(m, *args, **kw):
    """The ragged call, run a second time on a workspace whose every byte is 0xFF (a NaN pattern): the first call sizes it."""
    m(*_dev(args), ragged=True, **kw)
    torch.cuda.synchronize()
    m._ws.fill_(255)
    out = m(*_dev(args), ragged=True, **kw)
    torch.cuda.synchronize()
    return out


def _solo(m, batch, b, tf=None, frame=False, **kw):
    spk, texts, lens, _ = batch
    n = int(lens[b])
    args = [spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n]
    if tf is not None:
        mel_lens, p_t, e_t, d_t = tf
        cols = int(mel_lens[b]) if frame else n
        cut = lambda t: None if t is None else t[b:b + 1, :cols]
        args += [None, mel_lens[b:b + 1], int(mel_lens[b]), cut(p_t), cut(e_t), d_t[b:b + 1, :n]]
    return m(*_dev(args), ragged=False, **kw)


def _check_vs_solo(m, out, batch, tf=None, frame=False, **kw):
    """Every utterance of the ragged result `out` against its solo run; returns the solo results (None for an empty utterance)."""
    lens = batch[2]
    solos = []
    for b in range(len(lens)):
        n, ml = int(lens[b]), int(out[9][b])
        for i in (0, 1):
            assert torch.equal(out[i][b, ml:], torch.zeros_like(out[i][b, ml:])), (b, i)
        if ml == 0:                                        # nothing to decode alone: the utterance is silence, all zeros (checked above)
            solos.append(None)
            continue
        s = _solo(m, batch, b, tf, frame, **kw)
        assert int(s[9][0]) == ml, b
        cols = ml if frame else n
        for i in (2, 3):
            assert torch.equal(out[i][b, :cols], s[i][0, :cols]), (b, i)
        assert torch.equal(out[4][b, :n], s[4][0, :n]) and torch.equal(out[5][b, :n], s[5][0, :n]), b
        for i in (0, 1):
            g = out[i][b, :ml]
            assert torch.isfinite(g).all() and torch.equal(g, s[i][0]), (b, i, (g - s[i][0]).abs().max().item())
        solos.append(s)
    return solos


# ---------------------------------------------------------------------------------------------------------------- whole model
@pytest.mark.parametrize("mask", list(TC_MASKS))
def test_ragged_lj_mixed_lengths_equal_solo(lj_configs, mask):
    """LJSpeech, B = 16, 5..128 phonemes: utterances on both sides of the 128-frame attention backend split."""
    m, _ = _model(lj_configs, seed=41, tc_mask=TC_MASKS[mask])
    batch = synth.make_batch(16, 128, seed=42, min_len=5)
    out = _ragged(m, *batch)
    ml = out[9].cpu()
    assert int(ml.min()) < 128 <= int(ml.max())
    _check_vs_solo(m, out, batch)
    # padded token ids are not read: the same batch with garbage in the padding gives the same valid outputs
    spk, texts, lens, Lm = batch
    noisy = texts.clone()
    pad = torch.arange(Lm)[None, :] >= lens[:, None]
    noisy[pad] = torch.randint(1, 361, (int(pad.sum()),), generator=torch.Generator().manual_seed(5))
    out2 = _ragged(m, spk, noisy, lens, Lm)
    assert torch.equal(out2[9], out[9])
    for i in (0, 1, 2, 3, 4, 5):
        assert torch.equal(out2[i], out[i]), i             # padded columns / rows are zeros or masked in both


@pytest.mark.parametrize("mask", list(TC_MASKS))
def test_ragged_libri_full_size_equal_solo(libri_configs, mask):
    """configs[3] at full size: LibriTTS multi-speaker, B = 64, 64..256 phonemes, T > 1000 with members <= 1000 frames, so the
    batch uses the long position table while those members alone use the model's own one."""
    m, _ = _model(libri_configs, seed=43, tc_mask=TC_MASKS[mask])
    batch = synth.make_batch(64, 256, seed=11, n_speakers=904, min_len=64)
    out = _ragged(m, *batch)
    ml = out[9].cpu()
    assert int(ml.max()) > 1000 and int(ml.min()) <= 1000
    _check_vs_solo(m, out, batch)


@pytest.mark.parametrize("mask", list(TC_MASKS))
def test_ragged_lj_paper_frame_level_equal_solo(scratch, mask):
    """config/LJSpeech_paper: frame-level pitch / energy predictors on the expanded sequence, bounded by each utterance's frames."""
    from oracle.gen_golden import paper_state_dict
    pc, mc = configs.make_configs("LJSpeech_paper", scratch)
    m, _ = _model((pc, mc), seed=0, tc_mask=TC_MASKS[mask], sd=paper_state_dict(pc, mc, 44))
    batch = synth.make_batch(8, 96, seed=45, min_len=8)
    out = _ragged(m, *batch, p_control=1.1)
    assert out[2].shape == out[0].shape[:2]
    _check_vs_solo(m, out, batch, frame=True, p_control=1.1)


@pytest.mark.parametrize("mask", list(TC_MASKS))
def test_ragged_teacher_forced_edge_lengths(lj_configs, mask):
    """Teacher-forced mel lengths {0, 1, 127, 128, 129, 1001, T}: tile and backend edges, both position tables.  An utterance of
    0 frames comes out as zeros and changes nothing else; garbage in the padded targets changes no valid output."""
    m, _ = _model(lj_configs, seed=46, tc_mask=TC_MASKS[mask])
    T = 1300
    frames = [0, 1, 127, 128, 129, 1001, T]
    src = [10, 1, 30, 40, 50, 100, 120]
    spk, texts, _, Lm = synth.make_batch(len(src), max(src), seed=47)
    lens = torch.tensor(src)
    texts = texts * (torch.arange(Lm)[None, :] < lens[:, None])
    d_t = torch.zeros(len(src), Lm, dtype=torch.long)
    for b, (n, f) in enumerate(zip(src, frames)):
        d_t[b, :n] = f // n
        d_t[b, :f % n] += 1
    g = torch.Generator().manual_seed(48)
    p_t, e_t = torch.randn(len(src), Lm, generator=g), torch.randn(len(src), Lm, generator=g)
    mel_lens = torch.tensor(frames)
    assert torch.equal(d_t.sum(1), mel_lens)
    batch = (spk, texts, lens, Lm)
    out = _ragged(m, spk, texts, lens, Lm, None, mel_lens, T, p_t, e_t, d_t)
    assert torch.equal(out[9].cpu(), mel_lens)
    _check_vs_solo(m, out, batch, tf=(mel_lens, p_t, e_t, d_t))
    pad = torch.arange(Lm)[None, :] >= lens[:, None]
    texts2, d2, p2, e2 = texts.clone(), d_t.clone(), p_t.clone(), e_t.clone()
    texts2[pad] = 7
    d2[pad] = 1000
    p2[pad] = float("nan")
    e2[pad] = 1e30
    out2 = _ragged(m, spk, texts2, lens, Lm, None, mel_lens, T, p2, e2, d2)
    assert torch.equal(out2[9], out[9])
    for i in (0, 1):
        assert torch.equal(out2[i], out[i]), i
    for i in (2, 3, 4):
        assert torch.equal(out2[i][~pad.to(DEV)], out[i][~pad.to(DEV)]), i


def test_ragged_vs_oracle_alone(lj_configs, parity_log):
    """A ragged batch against the CPU oracle run on each utterance alone, with the flip protocol of test_gpu_model: durations must
    match except on a rounding boundary; if any decision flips, the mel is compared teacher-forced on the oracle's own decisions."""
    m, sd = _model(lj_configs, seed=49)
    spk, texts, lens, Lm = synth.make_batch(6, 64, seed=50, min_len=10)
    out = m(*_dev((spk, texts, lens, Lm)), ragged=True)
    refs = [O.fastspeech2_forward(sd, spk[b:b + 1], texts[b:b + 1, :int(n)], lens[b:b + 1], int(n)) for b, n in enumerate(lens)]
    flips = 0
    for b, r in enumerate(refs):
        n = int(lens[b])
        for l in (out[5][b, :n].cpu() != r[5][0]).nonzero().flatten().tolist():
            v = float(torch.exp(r[4][0, l].double()) - 1)
            assert abs(v - (int(v) + 0.5)) < 2e-4, (b, l, v)
            flips += 1
        assert max((out[i][b, :n].cpu() - r[i][0]).abs().max().item() for i in (2, 3, 4)) < 1e-4, b
        for i, nm in ((2, "pitch"), (3, "energy")):
            edges = sd[f"variance_adaptor.{nm}_bins"]
            diff = (torch.bucketize(out[i][b, :n].cpu(), edges) != torch.bucketize(r[i][0], edges)).nonzero().flatten()
            for l in diff.tolist():
                assert (edges - r[i][0, l]).abs().min().item() < 2e-5, (b, nm, l)
            flips += diff.numel()
    if flips:                                              # teacher-forced on the oracle's decisions, utterance by utterance
        B = len(lens)
        d_t = torch.zeros(B, Lm, dtype=torch.long)
        p_t, e_t = torch.zeros(B, Lm), torch.zeros(B, Lm)
        for b, r in enumerate(refs):
            n = int(lens[b])
            d_t[b, :n], p_t[b, :n], e_t[b, :n] = r[5][0].long(), r[2][0], r[3][0]
        mel_lens = d_t.sum(1)
        out = m(*_dev((spk, texts, lens, Lm, None, mel_lens, int(mel_lens.max()), p_t, e_t, d_t)), ragged=True)
        refs = [O.fastspeech2_forward(sd, spk[b:b + 1], texts[b:b + 1, :int(n)], lens[b:b + 1], int(n), None, mel_lens[b:b + 1],
                                      int(mel_lens[b]), p_t[b:b + 1, :int(n)], e_t[b:b + 1, :int(n)], d_t[b:b + 1, :int(n)])
                for b, n in enumerate(lens)]
    worst = 0.0
    for b, r in enumerate(refs):
        ml = int(r[9][0])
        assert int(out[9][b]) == ml
        for i in (0, 1):
            worst = max(worst, (out[i][b, :ml].cpu() - r[i][0]).abs().max().item())
    parity_log("fs2_ragged_vs_oracle_alone_lj_B6", mel=worst, decision_flips_at_boundaries=flips)
    assert worst < MEL_TOL, worst


def test_ragged_end_to_end_with_the_ragged_vocoder(lj_configs):
    """Ragged FastSpeech2 -> ragged Generator (and vocoder_infer(ragged=True)) equals the solo FastSpeech2 -> Generator chain."""
    from fastspeech2_b200 import dropin
    pc, mc = lj_configs
    m, _ = _model(lj_configs, seed=51)
    h = AttrDict(configs.HIFIGAN_CONFIG)
    gen = Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=52))
    gen.eval()
    gen.remove_weight_norm()
    gen = gen.to(DEV)
    batch = synth.make_batch(5, 48, seed=53, min_len=6)
    out = _ragged(m, *batch)
    hop = pc["preprocessing"]["stft"]["hop_length"]
    wav = gen(out[1].transpose(1, 2), mel_lens=out[9])
    wavs = dropin.vocoder_infer(out[1].transpose(1, 2), gen, mc, pc, lengths=out[9] * hop, ragged=True)
    for b in range(5):
        s = _solo(m, batch, b)
        ml = int(s[9][0])
        solo_wav = gen(s[1].transpose(1, 2))
        assert torch.equal(wav[b, :, :ml * 256], solo_wav[0]), b
        assert torch.equal(wav[b, :, ml * 256:], torch.zeros_like(wav[b, :, ml * 256:])), b
        want = dropin.vocoder_infer(s[1].transpose(1, 2), gen, mc, pc, lengths=s[9] * hop)[0]
        assert np.array_equal(wavs[b], want), b


# ---------------------------------------------------------------------------------------------------------------- operator
@pytest.mark.parametrize("taps,N,res", [(3, 256, False), (9, 1024, False), (1, 256, True)])
def test_segmented_conv_with_x_lens_equals_alone(taps, N, res):
    """The K-segmented tensor-core conv (FS2_TC_VARIANT_NB64 | SEGMENTED: encoder and predictor layers) with x_lens: every
    utterance's rows equal the same conv run on those rows alone, with NaN in every row beyond them and in the output."""
    B, T, Cin = 6, 700, 256
    lens = [0, 1, 127, 128, 129, T]
    g = torch.Generator().manual_seed(54)
    w = torch.randn(taps, Cin, N, generator=g) * 0.05
    bias = torch.randn(N, generator=g).to(DEV)
    x = torch.randn(B, T, Cin, generator=g)
    r = torch.randn(B, T, N, generator=g) if res else None
    for b, n in enumerate(lens):
        x[b, n:] = float("nan")
        if res:
            r[b, n:] = float("nan")
    x, r, wd = x.to(DEV), (r.to(DEV) if res else None), w.to(DEV)
    seg = packing.pack_conv_tc_segments(w).to(DEV)
    kw = dict(pad_left=(taps - 1) // 2, w_tc=seg, backend=L.CONV_TC, tc_variant=L.TC_VARIANT_NB64 | L.TC_VARIANT_SEGMENTED)
    if res:
        kw.update(in_act=L.ACT_LRELU, in_slope=0.0)
    out = torch.full((B, T, N), float("nan"), device=DEV)
    ops.conv1d(x, wd, bias, res=r, out=out, x_lens=torch.tensor(lens, dtype=torch.int32, device=DEV), **kw)
    for b, n in enumerate(lens):
        if n == 0:
            continue
        alone = ops.conv1d(x[b:b + 1, :n].contiguous(), wd, bias, res=None if r is None else r[b:b + 1, :n].contiguous(), **kw)
        assert torch.isfinite(out[b, :n]).all() and torch.equal(out[b, :n], alone[0]), (b, n)
