"""GPU: the acoustic voices mode (VoiceBank) with the eight voices of tests/voice_cases.py, which differ in every table and in every
tensor-core layer's weight-scale headers (segment headers of the K-segmented convs included), at the plans large batches pick.
  1. the PostNet's first conv at every channel-group size NG the planner gives it, in both operand formats, with voices mixed so that
     every persistent CTA's consecutive work items belong to different voices;
  2. every tc_mask policy of tests/test_gpu_acoustic_voices.py at a small batch and at an NG >= 2 batch;
  3. the exact kernels (tc_mask = 0) at batches that reach every (BM, BN) tile fs2_conv_simt_plan gives the acoustic convs;
  4. two utterances per voice of a large ragged batch against the CPU oracle on that voice's weights (the bit-equality bars cannot
     see an error that the solo and bank paths share);
  5. padded mode with a device voice index out of range.
The bar of 1, 2, 3 and 5 is torch.equal against each voice alone, as in tests/test_gpu_acoustic_voices.py; the batches of 1 and 3
fix their frame counts with d_targets, so the plan is known before the call."""
import pytest
import torch

from fastspeech2_b200 import synth
from fastspeech2_b200.model import FastSpeech2, VoiceBank
from tests import voice_cases as V
from tests.test_gpu_acoustic_voices import MASKS, _check_padded, _check_ragged, _dev
from tests.test_gpu_conv_groups import device_sms
from tests.test_gpu_model import _free_running_then_teacher_forced

pytestmark = pytest.mark.gpu
DEV = "cuda"
VOICE9 = [3, 0, 7, 1, 6, 2, 5, 4, 1]


def _models(cfgs, tc_mask=None):
    pc, mc = cfgs
    out = []
    for sd in V.voice_state_dicts(pc, mc):
        m = FastSpeech2(pc, mc)
        m.load_state_dict(sd)
        if tc_mask is not None:
            m.tc_mask = tc_mask
        out.append(m.to(DEV).eval())
    return out


def _check_forced(models, bank, voice, fb):
    """A teacher-forced batch (voice_cases.forced_batch), padded and ragged, bit for bit against each utterance's voice alone."""
    spk, texts, lens, Lm, mel_lens, d = fb
    T = int(mel_lens.max())
    out = _check_padded(models, bank, voice, (spk, texts, lens, Lm, None, mel_lens, T, None, None, d))
    assert out[0].shape[1] == T
    out = bank(torch.tensor(voice), *_dev([spk, texts, lens, Lm, None, mel_lens, T, None, None, d]), ragged=True)
    for b, k in enumerate(voice):
        n, ml = int(lens[b]), int(mel_lens[b])
        assert int(out[9][b]) == ml, b
        s = models[k](*_dev([spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n, None, mel_lens[b:b + 1], ml, None, None,
                             d[b:b + 1, :n]]), ragged=True)
        for i in (0, 1):
            assert torch.equal(out[i][b, :ml], s[i][0]), (b, i)
        for i in (2, 3, 4):
            assert torch.equal(out[i][b, :n], s[i][0, :n]), (b, i)


@pytest.mark.parametrize("target", V.GROUP_TARGETS, ids=lambda t: f"{t[0]}_ng{t[2]}")
def test_postnet_channel_groups_in_voices_mode(lj_configs, target):
    mask, fmt, NG, T = target
    B, plan, fb, voice = V.group_batch(fmt, NG, T, device_sms())
    assert plan["NG"] == NG and sorted(set(voice)) == list(range(V.MAX_VOICES)), (B, plan, voice)
    models = _models(lj_configs, MASKS[mask])
    _check_forced(models, VoiceBank(models), voice, fb)


@pytest.mark.parametrize("shape", ["small", "ng2"])
@pytest.mark.parametrize("mask", sorted(MASKS))
def test_segment_and_voice_headers(lj_configs, mask, shape):
    models = _models(lj_configs, MASKS[mask])
    bank = VoiceBank(models)
    if shape == "small":                               # free-running, 96 phonemes: every table within max_seq_len
        batch = synth.make_batch(len(VOICE9), 96, seed=91, min_len=6)
        _check_ragged(models, bank, VOICE9, batch)
        _check_padded(models, bank, VOICE9, batch)
    else:
        B, plan, fb, voice = V.group_batch("split3" if mask == "no_f8" else "f8", 2, V.GROUP_T, device_sms(), seed=92)
        _check_forced(models, bank, voice, fb)


def test_exact_path_reaches_every_simt_tile(lj_configs):
    _, mc = lj_configs
    sms = device_sms()
    want = V.simt_universe(mc, sms)
    assert V.simt_tiles(V.EXACT_SHAPES, mc, sms) == want, want
    models = _models(lj_configs, 0)
    bank = VoiceBank(models)
    for k, (B, L_, T) in enumerate(V.EXACT_SHAPES):
        fb = V.forced_batch(B, L_, T, seed=93 + k)
        assert int(fb[3]) == L_
        voice = [5] if B == 1 else [(3 * b + b // 8) % V.MAX_VOICES for b in range(B)]
        _check_forced(models, bank, voice, fb)


def test_bank_against_the_oracle(lj_configs, parity_log):
    """24 utterances of 48 to 96 phonemes, ragged: up to max_seq_len frames, so that every utterance reads its voice's own position
    tables as it would alone, and 7 or 8 tiles of 128 rows each, at which the PostNet's first conv plans NG >= 2.  Two utterances of
    each voice against the CPU oracle on that voice's state dict, by the flip-aware protocol of tests/test_gpu_model.py."""
    pc, mc = lj_configs
    sds = V.voice_state_dicts(pc, mc)
    models = _models(lj_configs)
    bank = VoiceBank(models)
    B = 24
    voice = [b % V.MAX_VOICES for b in range(B)]
    batch = synth.make_batch(B, 96, seed=94, min_len=48)
    out = bank(torch.tensor(voice), *_dev(batch), ragged=True)
    T = int(out[0].shape[1])
    assert T <= mc["max_seq_len"] and V.G.plan(V.postnet0_case("f8", 1, T), B, device_sms())["NG"] >= 2, T
    spk, texts, lens, _ = batch
    for b in range(2 * V.MAX_VOICES):
        k, n, ml = voice[b], int(lens[b]), int(out[9][b])

        def one(*a, **kw):
            if len(a) == 4 and not kw:                 # free-running: utterance b of the big batch's call
                cut = lambda i, t: t[b:b + 1, :ml] if i in (0, 1, 7) else (t[b:b + 1, :n] if i < 7 else t[b:b + 1])
                return tuple(cut(i, t) for i, t in enumerate(out))
            return bank(torch.tensor([k]), *a, ragged=True, **kw)     # teacher-forced on the oracle's decisions
        _free_running_then_teacher_forced(one, sds[k], (spk[b:b + 1], texts[b:b + 1, :n], lens[b:b + 1], n),
                                          f"voices_bank_vs_oracle_voice{k}_utt{b}", parity_log)


def test_padded_device_index_out_of_range_gives_an_empty_utterance(lj_configs):
    models = _models(lj_configs)
    bank = VoiceBank(models)
    batch = _dev(synth.make_batch(len(VOICE9), 64, seed=95, min_len=8))
    good = bank(torch.tensor(VOICE9, device=DEV), *batch, ragged=False)
    T = int(good[0].shape[1])
    bad_voice = list(VOICE9)
    bad_voice[2], bad_voice[6] = V.MAX_VOICES, -1
    bad = bank(torch.tensor(bad_voice, device=DEV), *batch, max_mel_len=T, ragged=False)
    assert bad[0].shape == good[0].shape
    for b in range(len(VOICE9)):
        if b in (2, 6):
            assert int(bad[9][b]) == 0 and not bad[5][b].any(), b
            continue
        for i in range(10):
            if torch.is_tensor(good[i]) and good[i].dim() > 0:
                assert torch.equal(bad[i][b], good[i][b]), (b, i)
