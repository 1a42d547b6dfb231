"""GPU: tensor-valued p_control / d_control through FastSpeech2.forward and fs2_acoustic_{encode,decode}_ctl.

  - a control tensor holding fp32(c) everywhere gives the scalar c's outputs bit for bit, whatever its shape, strides, dtype or device;
  - per-utterance ([B, 1]) and per-phoneme ([B, L]) controls against the CPU oracle and against the unmodified reference's outputs
    (tests/golden/fs2_controls.npz), with the flip-aware protocol of test_gpu_model;
  - ragged mode: utterance b with its slice of the controls equals its solo call, and control columns past its length are not read;
  - controls the reference never reads change nothing."""
import copy

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from fastspeech2_b200.model import FastSpeech2
from oracle import fs2_oracle as O
from tests.test_controls_cpu import load_case
from tests.test_gpu_model import _free_running_then_teacher_forced
from tests.test_gpu_ragged_acoustic import _check_vs_solo, _ragged

pytestmark = pytest.mark.gpu
DEV = "cuda"
MEL_TOL = 1e-3


def _model(cfgs, sd, tc_mask=None):
    m = FastSpeech2(*cfgs)
    m.load_state_dict(sd)
    if tc_mask is not None:
        m.tc_mask = tc_mask
    return m.to(DEV).eval()


def _paper(scratch, seed):
    from oracle.gen_golden import paper_state_dict
    pc, mc = configs.make_configs("LJSpeech_paper", scratch)
    return (pc, mc), paper_state_dict(pc, mc, seed)


def _frame_lj(scratch):
    pc, mc = configs.make_configs("LJSpeech", scratch)
    pc = copy.deepcopy(pc)
    pc["preprocessing"]["pitch"]["feature"] = "frame_level"
    pc["preprocessing"]["energy"]["feature"] = "frame_level"
    return pc, mc


def _controls(B, Lm, seed, per_phoneme):
    g = torch.Generator().manual_seed(seed)
    cols = Lm if per_phoneme else 1
    return 0.8 + 0.45 * torch.rand(B, cols, generator=g), 0.5 + 1.5 * torch.rand(B, cols, generator=g)


def _same(a, b):
    for i in (0, 1, 2, 3, 4, 5, 6, 7, 9):
        assert torch.equal(a[i], b[i]), i


# ---------------------------------------------------------------------------------------------------------------- 1. scalar equivalence
def _forms(c, shape):
    """fp32(c) as tensors of `shape` in every layout the normaliser takes: contiguous, [B, 1], stride-0 view, CPU, float64."""
    B = shape[0]
    return {"full": torch.full(shape, c, device=DEV), "per_utterance": torch.full((B, 1), c, device=DEV),
            "expanded": torch.full((1, 1), c, device=DEV).expand(shape), "cpu": torch.full(shape, c),
            "float64": torch.full(shape, c, dtype=torch.float64, device=DEV)}


@pytest.mark.parametrize("tc", ["default", "fp32_cuda_cores"])
@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("cfg", ["lj", "paper"])
def test_control_tensor_of_one_value_equals_the_scalar(cfg, ragged, tc, lj_configs, scratch):
    if cfg == "lj":
        cfgs, sd = lj_configs, synth.fastspeech2_state_dict(*lj_configs, seed=71)
    else:
        cfgs, sd = _paper(scratch, 72)
    m = _model(cfgs, sd, None if tc == "default" else 0)
    spk, texts, lens, Lm = synth.make_batch(4, 40, seed=73, min_len=9)
    args = [x.to(DEV) if torch.is_tensor(x) else x for x in (spk, texts, lens, Lm)]
    pc, dc = float(np.float32(1.1)), float(np.float32(1.3))
    want = m(*args, p_control=pc, d_control=dc, ragged=ragged)
    B = len(lens)
    p_shape = (B, Lm) if cfg == "lj" else (B, 1)           # frame-level p broadcasts to [B, T]: per-utterance only
    for (kp, p), (kd, d) in zip(_forms(pc, p_shape).items(), _forms(dc, (B, Lm)).items()):
        got = m(*args, p_control=p, d_control=d, ragged=ragged)
        _same(got, want)
        _same(m(*args, p_control=p, d_control=dc, ragged=ragged), want)
        _same(m(*args, p_control=pc, d_control=d, ragged=ragged), want)


# ---------------------------------------------------------------------------------------------------------------- 2. against the oracle
@pytest.mark.parametrize("per_phoneme", [False, True])
@pytest.mark.parametrize("cfg", ["lj_B16_L128", "libri_B6_L64-256"])
def test_controls_against_the_oracle(cfg, per_phoneme, lj_configs, libri_configs, parity_log):
    if cfg.startswith("lj"):
        cfgs, batch = lj_configs, synth.make_batch(16, 128, seed=75)
    else:
        cfgs, batch = libri_configs, synth.make_batch(6, 256, seed=76, n_speakers=904, min_len=64)
    sd = synth.fastspeech2_state_dict(*cfgs, seed=74)
    m = _model(cfgs, sd)
    p, d = _controls(len(batch[2]), batch[3], 77, per_phoneme)
    out, ref = _free_running_then_teacher_forced(m, sd, batch, f"fs2_controls_{cfg}_{'phoneme' if per_phoneme else 'utterance'}",
                                                 parity_log, p_control=p, d_control=d)
    plain = O.fastspeech2_decisions(sd, *batch)
    assert not torch.equal(plain[3], ref[5])               # the controls changed the durations


# ---------------------------------------------------------------------------------------------------------------- 3. golden
@pytest.mark.parametrize("name", ["lj_utt", "lj_phoneme", "libri_utt", "paper_utt_phoneme"])
def test_controls_against_the_reference_outputs(name, scratch, parity_log):
    cfgs, sd, inputs, ctl, want, frame = load_case(name, scratch)
    m = _model(cfgs, sd)
    spk, texts, lens, Lm = inputs
    lv = dict(pitch_level="frame_level", energy_level="frame_level") if frame else {}
    T = int(want[9].max())
    forced = O.fastspeech2_forward(sd, spk, texts, lens, Lm, None, want[9], T, want[2], want[3], want[5].long(), **ctl, **lv)
    _free_running_then_teacher_forced(m, sd, inputs, f"fs2_controls_golden_{name}", parity_log, oracle=(want, forced), raw_heads=frame,
                                      **ctl)


# ---------------------------------------------------------------------------------------------------------------- 4. ragged
def _check_each_vs_solo(m, out, batch, kw_of, frame=False):
    spk, texts, lens, Lm = batch
    for b in range(len(lens)):
        one = tuple(x[b:b + 1] if torch.is_tensor(x) else x for x in out)
        _check_vs_solo(m, one, (spk[b:b + 1], texts[b:b + 1], lens[b:b + 1], Lm), frame=frame, **kw_of(b, int(lens[b])))


@pytest.mark.parametrize("per_phoneme", [False, True])
@pytest.mark.parametrize("tc", ["default", "fp32_cuda_cores"])
def test_ragged_controls_equal_solo(tc, per_phoneme, lj_configs):
    """Utterance b equals its solo call with c[b] ([B, 1]) or c[b:b+1, :src_lens[b]] ([B, L]).  Control columns past src_lens[b]
    hold NaN: one read would show in that utterance's outputs."""
    m = _model(lj_configs, synth.fastspeech2_state_dict(*lj_configs, seed=78), None if tc == "default" else 0)
    batch = synth.make_batch(10, 96, seed=79, min_len=5)
    lens = batch[2]
    p, d = _controls(len(lens), batch[3], 80, per_phoneme)
    if per_phoneme:
        pad = torch.arange(batch[3])[None, :] >= lens[:, None]
        p[pad], d[pad] = float("nan"), float("nan")
    out = _ragged(m, *batch, p_control=p.to(DEV), d_control=d.to(DEV))
    if per_phoneme:
        kw_of = lambda b, n: dict(p_control=p[b:b + 1, :n].to(DEV), d_control=d[b:b + 1, :n].to(DEV))
    else:
        kw_of = lambda b, n: dict(p_control=float(p[b, 0]), d_control=float(d[b, 0]))
    _check_each_vs_solo(m, out, batch, kw_of)


def test_ragged_frame_level_per_utterance_control_equals_solo(scratch):
    """LJSpeech_paper: frame-level pitch / energy scaled per utterance; frames past mel_lens[b] are not read."""
    cfgs, sd = _paper(scratch, 81)
    m = _model(cfgs, sd)
    batch = synth.make_batch(6, 64, seed=82, min_len=6)
    p, d = _controls(6, 64, 83, False)
    out = _ragged(m, *batch, p_control=p.to(DEV), d_control=d.to(DEV))
    _check_each_vs_solo(m, out, batch, lambda b, n: dict(p_control=float(p[b, 0]), d_control=float(d[b, 0])), frame=True)


# ---------------------------------------------------------------------------------------------------------------- 5. frame level
def test_frame_level_per_frame_control_with_fixed_frames(scratch, parity_log):
    """A [B, T] p_control for frame-level predictors, T fixed by max_mel_len and d_targets; a [B, L] one raises ValueError."""
    cfgs = _frame_lj(scratch)
    sd = synth.fastspeech2_state_dict(*cfgs, seed=84)
    m = _model(cfgs, sd)
    spk, texts, lens, Lm = synth.make_batch(4, 40, seed=85, min_len=20)
    lv = dict(pitch_level="frame_level", energy_level="frame_level")
    d_t = O.fastspeech2_forward(sd, spk, texts, lens, Lm, **lv)[5].long()
    mel_lens = d_t.sum(1)
    T = int(mel_lens.max())
    p = 0.8 + 0.45 * torch.rand(4, T, generator=torch.Generator().manual_seed(86))
    tf = (None, mel_lens, T, None, None, d_t)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm, *tf, p_control=p, **lv)
    dev = lambda xs: [x.to(DEV) if torch.is_tensor(x) else x for x in xs]
    out = m(*dev((spk, texts, lens, Lm) + tf), p_control=p.to(DEV))
    e = {nm: (out[i].cpu() - ref[i]).abs().max().item() for i, nm in ((2, "pitch"), (3, "energy"))}
    assert max(e.values()) < 1e-4, e
    flips = 0
    for i, nm in ((2, "pitch"), (3, "energy")):
        edges = sd[f"variance_adaptor.{nm}_bins"]
        diff = (torch.bucketize(out[i].cpu(), edges) != torch.bucketize(ref[i], edges)).nonzero()
        for b, t in diff.tolist():
            assert (edges - ref[i][b, t]).abs().min().item() < 2e-5, (nm, b, t)
        flips += diff.shape[0]
    if flips:                                              # a bucket on an edge: compare the mel on the oracle's own decisions
        tf = (None, mel_lens, T, ref[2], ref[3], d_t)
        ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm, *tf, p_control=p, **lv)
        out = m(*dev((spk, texts, lens, Lm) + tf), p_control=p.to(DEV))
    e.update(mel=(out[0].cpu() - ref[0]).abs().max().item(), postnet=(out[1].cpu() - ref[1]).abs().max().item())
    parity_log("fs2_controls_frame_level_per_frame", **e, decision_flips_at_boundaries=flips)
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL, e
    with pytest.raises(ValueError, match="p_control"):
        m(*dev((spk, texts, lens, Lm)), p_control=torch.ones(4, Lm, device=DEV))


# ---------------------------------------------------------------------------------------------------------------- 6. ignored controls
def test_controls_the_reference_never_reads_change_nothing(lj_configs):
    sd = synth.fastspeech2_state_dict(*lj_configs, seed=87)
    m = _model(lj_configs, sd)
    spk, texts, lens, Lm = synth.make_batch(3, 30, seed=88, min_len=12)
    args = [x.to(DEV) if torch.is_tensor(x) else x for x in (spk, texts, lens, Lm)]
    want = m(*args, e_control=1.0)
    for e in (torch.rand(7, device=DEV), torch.rand(2, 3, 4), torch.rand(3, 30, 1, dtype=torch.float64), "anything", None):
        _same(m(*args, e_control=e), want)
    free = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    tf = [free[9], int(free[9].max()), free[2], free[3], free[5].long()]
    tf_args = args + [None] + [x.to(DEV) if torch.is_tensor(x) else x for x in tf]
    want = m(*tf_args)
    for c in (torch.rand(5, 7, 9, device=DEV), torch.rand(3, 30, 1), "anything"):
        _same(m(*tf_args, p_control=c, d_control=c, e_control=c), want)


# ---------------------------------------------------------------------------------------------------------------- 7. end to end
def test_ragged_controls_end_to_end_with_the_vocoder(lj_configs):
    """Ragged FastSpeech2 with per-utterance controls -> Generator(mel, mel_lens): every waveform equals its solo synthesis."""
    m = _model(lj_configs, synth.fastspeech2_state_dict(*lj_configs, seed=89))
    h = AttrDict(configs.HIFIGAN_CONFIG)
    gen = Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=90))
    gen.eval()
    gen.remove_weight_norm()
    gen = gen.to(DEV)
    spk, texts, lens, Lm = synth.make_batch(5, 48, seed=91, min_len=6)
    p, d = _controls(5, Lm, 92, False)
    out = _ragged(m, spk, texts, lens, Lm, p_control=p.to(DEV), d_control=d.to(DEV))
    wav = gen(out[1].transpose(1, 2), mel_lens=out[9])
    for b in range(5):
        n = int(lens[b])
        s = m(spk[b:b + 1].to(DEV), texts[b:b + 1, :n].to(DEV), lens[b:b + 1].to(DEV), n, p_control=float(p[b, 0]),
              d_control=float(d[b, 0]))
        ml = int(s[9][0])
        assert int(out[9][b]) == ml
        assert torch.equal(wav[b, :, :ml * 256], gen(s[1].transpose(1, 2))[0]), b
        assert torch.equal(wav[b, :, ml * 256:], torch.zeros_like(wav[b, :, ml * 256:])), b
