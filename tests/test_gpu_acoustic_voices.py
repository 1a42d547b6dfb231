"""GPU: several FastSpeech2 voices in one acoustic call (VoiceBank, fs2_acoustic_{encode,decode}_voices), bit for bit against each
utterance's own voice.  The bar is torch.equal throughout: the plan is voice 0's, no kernel mixes batch rows, and only where each
utterance reads its weights and tables from changes.
  * ragged: utterance b equals models[voice[b]] called alone on its slice (ragged=True);
  * padded: row b of every output equals row b of models[voice[b]] on the whole batch with max_mel_len = T of the bank's call."""
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.model import FastSpeech2, VoiceBank

pytestmark = pytest.mark.gpu
DEV = "cuda"
ALL = L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8 | L.TC_ENCODER | L.TC_PREDICTORS
MASKS = {"default": None, "exact": 0, "no_f8": L.TC_DECODER | L.TC_POSTNET | L.TC_ENCODER | L.TC_PREDICTORS,
         "exact_encoder": L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8}
VOICE = [0, 2, 1, 1, 0, 2, 1]


def _voice(cfgs, seed, tc_mask=None, sd=None, bins=1.0):
    """A voice: a FastSpeech2 from a synthetic seed; bins != 1 scales its pitch / energy bins (a voice with other stats.json)"""
    pc, mc = cfgs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=seed) if sd is None else dict(sd)
    if bins != 1.0:
        for k in ("variance_adaptor.pitch_bins", "variance_adaptor.energy_bins"):
            sd[k] = sd[k] * bins
    m = FastSpeech2(pc, mc)
    m.load_state_dict(sd)
    if tc_mask is not None:
        m.tc_mask = tc_mask
    return m.to(DEV).eval()


def _voices(cfgs, tc_mask=None, seeds=(51, 52, 53)):
    return [_voice(cfgs, s, tc_mask, bins=1.07 if k == 2 else 1.0) for k, s in enumerate(seeds)]


def _dev(xs):
    return [x.to(DEV) if torch.is_tensor(x) else x for x in xs]


def _check_padded(models, bank, voice, args, **kw):
    out = bank(torch.tensor(voice), *_dev(args), ragged=False, **kw)
    T = out[0].shape[1]
    full = list(args) + [None] * (10 - len(args))
    full[6] = T                                        # max_mel_len
    for k in sorted(set(voice)):
        ref = models[k](*_dev(full), ragged=False, **kw)
        for b in (b for b, v in enumerate(voice) if v == k):
            for i in range(10):
                if torch.is_tensor(out[i]) and out[i].dim() > 0:
                    assert torch.equal(out[i][b], ref[i][b]), (b, k, i)
    return out


def _check_ragged(models, bank, voice, batch, **kw):
    out = bank(torch.tensor(voice), *_dev(batch), ragged=True, **kw)
    spk, texts, lens, _ = batch
    for b, k in enumerate(voice):
        n, ml = int(lens[b]), int(out[9][b])
        s = models[k](*_dev([spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n]), ragged=True, **_slice_ctl(kw, b, n))
        assert int(s[9][0]) == ml, b
        for i in (0, 1):
            assert torch.equal(out[i][b, :ml], s[i][0]), (b, i)
        for i in (2, 3, 4, 5):
            assert torch.equal(out[i][b, :n], s[i][0, :n]), (b, i)
    return out


def _slice_ctl(kw, b, n):
    cut = lambda c: c[b:b + 1, :n] if torch.is_tensor(c) and c.dim() == 2 and c.shape[1] > 1 else (c[b:b + 1] if torch.is_tensor(c) else c)
    return {k: cut(v) for k, v in kw.items()}


@pytest.mark.parametrize("mask", sorted(MASKS))
def test_three_lj_voices_equal_each_voice(lj_configs, mask):
    models = _voices(lj_configs, MASKS[mask])
    bank = VoiceBank(models)
    batch = synth.make_batch(len(VOICE), 96, seed=54, min_len=6)
    _check_ragged(models, bank, VOICE, batch)
    _check_padded(models, bank, VOICE, batch)


def test_libri_per_utterance_speakers(libri_configs):
    models = _voices(libri_configs)
    bank = VoiceBank(models)
    batch = synth.make_batch(len(VOICE), 80, seed=55, n_speakers=904, min_len=10)
    _check_ragged(models, bank, VOICE, batch)
    _check_padded(models, bank, VOICE, batch)


def test_lj_paper_frame_level(scratch):
    from oracle.gen_golden import paper_state_dict
    pc, mc = configs.make_configs("LJSpeech_paper", scratch)
    models = [_voice((pc, mc), 0, sd=paper_state_dict(pc, mc, s), bins=1.07 if s == 58 else 1.0) for s in (56, 57, 58)]
    bank = VoiceBank(models)
    batch = synth.make_batch(len(VOICE), 64, seed=59, min_len=8)
    _check_padded(models, bank, VOICE, batch, p_control=1.1)
    out = bank(torch.tensor(VOICE), *_dev(batch), ragged=True, p_control=1.1)
    assert out[2].shape == out[0].shape[:2]


def test_controls_and_teacher_forcing(lj_configs):
    models = _voices(lj_configs)
    bank = VoiceBank(models)
    spk, texts, lens, Lm = synth.make_batch(len(VOICE), 64, seed=60, min_len=8)
    g = torch.Generator().manual_seed(61)
    p_u = 0.8 + 0.4 * torch.rand(len(VOICE), 1, generator=g)
    d_p = 0.7 + 0.6 * torch.rand(len(VOICE), Lm, generator=g)
    _check_ragged(models, bank, VOICE, (spk, texts, lens, Lm), p_control=p_u, d_control=d_p)
    _check_padded(models, bank, VOICE, (spk, texts, lens, Lm), p_control=p_u, d_control=d_p)
    d_t = torch.randint(0, 6, (len(VOICE), Lm), generator=g) * (torch.arange(Lm)[None] < lens[:, None])
    mel_lens = d_t.sum(1)
    T = int(mel_lens.max())
    p_t, e_t = torch.randn(len(VOICE), Lm, generator=g), torch.randn(len(VOICE), Lm, generator=g)
    _check_padded(models, bank, VOICE, (spk, texts, lens, Lm, None, mel_lens, T, p_t, e_t, d_t))


def test_one_voice_bank_equals_forward_and_launch_counts(lj_configs):
    models = _voices(lj_configs)
    batch = _dev(synth.make_batch(5, 80, seed=62, min_len=6))
    for ragged in (False, True):
        ref = models[0](*batch, ragged=ragged)
        out = VoiceBank(models[:1])(torch.zeros(5, dtype=torch.long), *batch, ragged=ragged)
        for i in range(10):
            if torch.is_tensor(ref[i]):
                assert torch.equal(out[i], ref[i]), (ragged, i)
    T = int(ref[0].shape[1])
    lib = L.lib()

    def launches(fn):
        fn()                                           # warm (packing, workspaces)
        torch.cuda.synchronize()
        n0 = lib.fs2_kernel_launch_count()
        fn()
        torch.cuda.synchronize()
        return lib.fs2_kernel_launch_count() - n0
    for ragged in (False, True):
        base = launches(lambda: models[0](*batch, ragged=ragged, max_mel_len=T))
        for n in (1, 2, 3):
            voice = torch.tensor([k % n for k in range(5)])
            assert launches(lambda: VoiceBank(models[:n])(voice, *batch, ragged=ragged, max_mel_len=T)) == base, (ragged, n)


def test_device_index_out_of_range_gives_an_empty_utterance(lj_configs):
    models = _voices(lj_configs)
    bank = VoiceBank(models)
    batch = _dev(synth.make_batch(len(VOICE), 64, seed=63, min_len=8))
    good = bank(torch.tensor(VOICE, device=DEV), *batch, ragged=True)
    bad_voice = list(VOICE)
    bad_voice[3], bad_voice[5] = 7, -1
    bad = bank(torch.tensor(bad_voice, device=DEV), *batch, ragged=True)
    for b in range(len(VOICE)):
        if b in (3, 5):
            assert int(bad[9][b]) == 0 and not bad[5][b].any(), b
            continue
        ml, n = int(good[9][b]), int(batch[2][b])
        assert int(bad[9][b]) == ml
        for i in (0, 1):
            assert torch.equal(bad[i][b, :ml], good[i][b, :ml]), (b, i)
        for i in (2, 3, 4, 5):
            assert torch.equal(bad[i][b, :n], good[i][b, :n]), (b, i)


def test_side_stream_equals_default_stream(lj_configs):
    models = _voices(lj_configs)
    bank = VoiceBank(models)
    batch = _dev(synth.make_batch(len(VOICE), 64, seed=64, min_len=8))
    voice = torch.tensor(VOICE, device=DEV)
    ref = bank(voice, *batch, ragged=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        out = bank(voice, *batch, ragged=True)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for i in range(10):
        if torch.is_tensor(ref[i]):
            assert torch.equal(out[i], ref[i]), i


def test_end_to_end_into_a_multi_generator_pool(lj_configs):
    from tests.test_gpu_stream_multi import _run
    from tests.test_gpu_stream_vocoder import _generator
    models = _voices(lj_configs)
    bank = VoiceBank(models)
    gens = [_generator(configs.HIFIGAN_CONFIG, seed=s) for s in (3, 11, 17)]
    batch = _dev(synth.make_batch(len(VOICE), 48, seed=65, min_len=8))
    out = bank(torch.tensor(VOICE), *batch, ragged=True)
    mels = [out[1][b, :int(out[9][b])].transpose(0, 1).contiguous() for b in range(len(VOICE))]
    pool = gens[0].stream_pool(chunk_frames=32, generators=gens[1:])
    wav = _run(pool, mels, VOICE, [0] * len(VOICE))
    spk, texts, lens, _ = batch
    for b, k in enumerate(VOICE):
        n = int(lens[b])
        alone = models[k](spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n, ragged=True)
        assert torch.equal(wav[b], gens[k](alone[1].transpose(1, 2))), b
