"""GPU: the two drop-in modules against the CPU oracle on identical inputs and weights.

Protocol (SURVEY.md section 7, hard part 2): (A) free-running -- continuous predictions are compared and the discrete
decisions (durations, hence mel_lens) must match exactly; (B) teacher-forced with the oracle's own decisions so a
boundary flip cannot hide or fake a mel error.  Bars from BASELINE.json: mel 1e-3, waveform 1e-4 max-abs."""
import numpy as np
import pytest
import torch

from fastspeech2_b200 import configs, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from fastspeech2_b200.model import FastSpeech2
from oracle import fs2_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda"
MEL_TOL, WAV_TOL = 1e-3, 1e-4


def _model(cfgs, seed):
    pc, mc = cfgs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=seed)
    m = FastSpeech2(pc, mc)
    m.load_state_dict(sd)
    return m.to(DEV).eval(), sd


def _cmp(out, ref):
    errs = {}
    for i, name in ((0, "mel"), (1, "postnet"), (2, "pitch"), (3, "energy"), (4, "logd")):
        errs[name] = (out[i].cpu() - ref[i]).abs().max().item()
    return errs


def _free_running_then_teacher_forced(m, sd, batch, name, parity_log, oracle=None, mel_tol=MEL_TOL, raw_heads=False, **kw):
    """SURVEY.md section 7, hard part 2: pitch / energy buckets are discrete decisions -- a prediction that lies within fp32 summation
    noise (~3e-6) of one of the 255 bin edges can land in different buckets on the GPU and in the CPU oracle (with ~10^4 phonemes
    per batch that happens for roughly one batch in four; the reference itself flips between thread counts), which swaps an
    embedding row and changes that utterance's whole mel.  Protocol: (A) free-running -- durations exact, continuous predictions
    within 1e-4, every bucket difference must be such a boundary case (margin < 2e-5) and is logged; (B) if any bucket differs, the
    mel is compared teacher-forced on the oracle's own decisions (p / e / d targets), which cannot hide a real error.  The same holds
    for a duration that sits on a rounding boundary of round(exp(logd) - 1) (margin < 2e-4 frames).  oracle: the oracle's free-running
    and teacher-forced outputs for this batch when the caller has them already.  raw_heads: pitch / energy are unnormalised (Hz and
    energy in the hundreds, config/LJSpeech_paper), so their bar (5e-4) and their bin-edge margin are relative to 1 + |oracle value|."""
    spk, texts, lens, Lm = batch
    dev = lambda t: t.to(DEV)
    ref = oracle[0] if oracle else O.fastspeech2_forward(sd, spk, texts, lens, Lm, **kw)
    out = m(dev(spk), dev(texts), dev(lens), Lm, **kw)
    flips = 0
    for b, l in (out[5].cpu() != ref[5]).nonzero().tolist():          # a duration on a rounding boundary (round-half-even of exp(logd) - 1)
        v = float(torch.exp(ref[4][b, l].double()) - 1)
        margin = abs(v - (int(v) + 0.5))
        assert margin < 2e-4, f"duration differs away from a rounding boundary: utterance {b} phoneme {l} exp(logd)-1 = {v}"
        flips += 1
    if not flips:
        assert torch.equal(out[9].cpu(), ref[9]) and torch.equal(out[7].cpu(), ref[7])
    unit = lambda r: 1 + r.abs() if raw_heads else 1.0
    err = lambda o, r: ((o.cpu() - r).abs() / unit(r)).max().item()
    # raw-valued heads: the fp32 noise the 100-250x head weights amplify is ~2e-4 of 1 + |value| (the relative bar of the paper config's
    # golden test), so a bucket may differ wherever the oracle's value lies within that of an edge
    cont_tol, edge_tol = (5e-4, 5e-4) if raw_heads else (1e-4, 2e-5)
    e = {"logd": (out[4].cpu() - ref[4]).abs().max().item()}
    assert e["logd"] < 1e-4, e
    # Each decision changes what the later predictors see: the energy predictor's input holds the pitch embedding, and frame-level
    # predictors run on the duration-expanded sequence.  So a prediction is compared free-running only while every decision before it
    # matched; after a boundary flip it is compared teacher-forced, where its input is the oracle's again.
    same_inputs = not flips or ref[2].shape == texts.shape
    for i, nm in ((2, "pitch"), (3, "energy")):
        if not same_inputs:
            break
        e[nm] = err(out[i], ref[i])
        assert e[nm] < cont_tol, e
        edges = sd[f"variance_adaptor.{nm}_bins"]
        bo, br = torch.bucketize(out[i].cpu(), edges), torch.bucketize(ref[i], edges)
        diff = (bo != br).nonzero()
        for b, l in diff.tolist():
            margin = ((edges - ref[i][b, l]).abs().min() / unit(ref[i][b, l])).item()
            assert margin < edge_tol, f"{nm} bucket differs away from a bin edge: utterance {b} position {l} margin {margin}"
        flips += diff.shape[0]
        same_inputs = diff.shape[0] == 0
    e_free = e
    if flips:
        T = int(ref[9].max())
        ref = oracle[1] if oracle else O.fastspeech2_forward(sd, spk, texts, lens, Lm, None, ref[9], T, ref[2], ref[3], ref[5].long(), **kw)
        out = m(dev(spk), dev(texts), dev(lens), Lm, None, dev(ref[9]), T, dev(ref[2]), dev(ref[3]), dev(ref[5].long()), **kw)
        e_tf = {nm: err(out[i], ref[i]) for i, nm in ((2, "pitch"), (3, "energy"))}
        assert max(e_tf.values()) < cont_tol, e_tf
    e = _cmp(out, ref)
    parity_log(name, **e, **{f"free_running_{k}": v for k, v in e_free.items()}, decision_flips_at_boundaries=flips, tmax=int(ref[9].max()),
               frames=int(ref[9].sum()))
    assert e["mel"] < mel_tol and e["postnet"] < mel_tol, e
    return out, ref


@pytest.mark.parametrize("B,L,min_len", [(1, 24, None), (3, 40, 17), (16, 128, None)])
def test_fastspeech2_free_running_lj(lj_configs, B, L, min_len, parity_log):
    m, sd = _model(lj_configs, seed=1)
    spk, texts, lens, Lm = synth.make_batch(B, L, seed=2, min_len=min_len)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm)
    assert torch.equal(out[5].cpu(), ref[5]), "duration decisions differ"
    assert torch.equal(out[9].cpu(), ref[9]) and torch.equal(out[6].cpu(), ref[6]) and torch.equal(out[7].cpu(), ref[7])
    e = _cmp(out, ref)
    parity_log(f"fs2_free_running_lj_B{B}_L{L}", **e)
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL and max(e["pitch"], e["energy"], e["logd"]) < 1e-4, e


def test_fastspeech2_multispeaker_controls(libri_configs, parity_log):
    m, sd = _model(libri_configs, seed=3)
    spk, texts, lens, Lm = synth.make_batch(5, 64, seed=4, n_speakers=904, min_len=20)
    kw = dict(p_control=1.15, e_control=0.8, d_control=1.3)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm, **kw)
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm, **kw)
    assert torch.equal(out[5].cpu(), ref[5]) and torch.equal(out[9].cpu(), ref[9])
    e = _cmp(out, ref)
    parity_log("fs2_multispeaker_controls_B5_L64", **e)
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL, e


def test_fastspeech2_ragged_multispeaker_long(libri_configs, parity_log):
    """BASELINE.json configs[3] in miniature: LibriTTS multi-speaker, mixed 64-256 phonemes with padding masks -> T up to ~2000
    (position table beyond max_seq_len, decoder attention with 2048 padded keys)."""
    m, sd = _model(libri_configs, seed=13)
    spk, texts, lens, Lm = synth.make_batch(6, 256, seed=14, n_speakers=904, min_len=64)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm)
    assert torch.equal(out[5].cpu(), ref[5]) and torch.equal(out[9].cpu(), ref[9]) and torch.equal(out[7].cpu(), ref[7])
    assert int(ref[9].max()) > 1500
    e = _cmp(out, ref)
    parity_log("fs2_ragged_libri_B6_L64-256", **e, tmax=int(ref[9].max()))
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL, e


def test_fastspeech2_full_size_vs_oracle(libri_configs, parity_log):
    """BASELINE.json configs[3] at FULL size (LibriTTS multi-speaker, B = 64, mixed 64-256 phonemes with padding masks, Tmax ~ 2000)
    against the CPU oracle on the whole batch (tens of seconds of ATen on the box's cores): decisions exact, mel within the bar,
    padded rows follow the reference's padding semantics.  Exercises many 128-row tiles per utterance, Tk > 1000 attention and the long position table."""
    pc, mc = libri_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=21)
    m = FastSpeech2(pc, mc); m.load_state_dict(sd); m = m.to(DEV).eval()
    batch = synth.make_batch(64, 256, seed=22, n_speakers=904, min_len=64)
    a, ref = _free_running_then_teacher_forced(m, sd, batch, "fs2_full_size_libri_B64_vs_oracle", parity_log)
    assert int(ref[9].max()) > 1800 and a[0].shape[0] == 64
    # padded mel rows equal mel_linear.bias exactly (decoder output is zeroed there, SURVEY.md App. A.7)
    bias = sd["mel_linear.bias"].to(DEV)
    pad = a[7]                                             # True = padded frame
    assert pad.any() and (a[0][pad] - bias).abs().max().item() < 1e-6
    assert torch.isfinite(a[1]).all()


def test_fastspeech2_config4_shard_vs_oracle(lj_configs, parity_log):
    """BASELINE.json configs[4]: one GPU's shard of the B = 512 job = a 64-utterance micro-batch of 128-phoneme LJSpeech inputs
    (-> ~1012 frames each), FastSpeech2 against the oracle on the whole micro-batch; its vocoder half is checked below."""
    m, sd = _model(lj_configs, seed=0)
    _free_running_then_teacher_forced(m, sd, synth.make_batch(64, 128, seed=3), "fs2_config4_shard_B64_L128_vs_oracle", parity_log)


@pytest.mark.parametrize("cfg", ["lj", "libri"])
def test_fastspeech2_tensor_core_encoder_and_predictors(cfg, lj_configs, libri_configs, parity_log):
    """Both settings of FS2_TC_ENCODER | FS2_TC_PREDICTORS (default: set): encoder FFT blocks and the three variance predictors on tensor-core, K-SEGMENTED (every
    (tap, 256-channel) slice its own 16-step accumulation, slices summed in fp32 by the epilogue) so that the truncating tensor-core
    accumulator cannot move the discrete decisions more than the fp32 kernels do.  Same flip-aware protocol as the full-size tests."""
    from fastspeech2_b200 import _lib as L
    pc, mc = lj_configs if cfg == "lj" else libri_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=31)
    batch = synth.make_batch(16, 128, seed=32, n_speakers=904 if cfg == "libri" else 1, min_len=40 if cfg == "libri" else None)
    for label, bits in (("tc_segmented", L.TC_ENCODER | L.TC_PREDICTORS), ("fp32_cuda_cores", 0)):
        m = FastSpeech2(pc, mc); m.load_state_dict(sd)
        m.tc_mask = (m.tc_mask & ~(L.TC_ENCODER | L.TC_PREDICTORS)) | bits
        m = m.to(DEV).eval()
        _free_running_then_teacher_forced(m, sd, batch, f"fs2_encoder_predictors_{label}_{cfg}_B16_L128", parity_log)


def test_fastspeech2_paper_config_golden(scratch, parity_log):
    """config/LJSpeech_paper (4-layer decoder, frame-level unnormalised pitch / energy, LOG-spaced pitch edges, model/modules.py:48-54)
    against the committed outputs of the unmodified reference (tests/golden/fs2_lj_paper.npz) and the oracle."""
    import numpy as np, os
    from oracle.gen_golden import paper_state_dict
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "fs2_lj_paper.npz"))
    pc, mc = configs.make_configs("LJSpeech_paper", scratch)
    sd = paper_state_dict(pc, mc, int(z["seed"]))
    m = FastSpeech2(pc, mc); m.load_state_dict(sd); m = m.to(DEV).eval()
    t = lambda k: torch.from_numpy(z[k])
    out = m(t("speakers").to(DEV), t("texts").to(DEV), t("src_lens").to(DEV), int(z["max_src_len"]), p_control=float(z["p_control"]))
    assert torch.equal(out[9].cpu(), t("mel_lens")) and torch.equal(out[5].cpu(), t("d_rounded")) and torch.equal(out[7].cpu(), t("mel_masks"))
    e = {"mel": (out[0].cpu() - t("mel")).abs().max().item(), "postnet": (out[1].cpu() - t("postnet_mel")).abs().max().item(),
         "pitch_rel": ((out[2].cpu() - t("p_pred")).abs() / (1 + t("p_pred").abs())).max().item(),
         "energy_rel": ((out[3].cpu() - t("e_pred")).abs() / (1 + t("e_pred").abs())).max().item()}
    edges = sd["variance_adaptor.pitch_bins"]
    same_bucket = torch.equal(torch.bucketize(out[2].cpu() , edges), torch.bucketize(t("p_pred"), edges))
    parity_log("fs2_lj_paper_golden", **e, same_pitch_buckets=float(same_bucket))
    # the raw-valued heads (weights x100..250, outputs in the hundreds) amplify fp32 summation noise: relative bar 5e-4
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL and e["pitch_rel"] < 5e-4 and e["energy_rel"] < 5e-4, e


def test_fastspeech2_frame_level_variances(scratch, parity_log):
    """pitch / energy feature = frame_level (config/LJSpeech_paper): predictors run on the expanded sequence."""
    import copy
    pc, mc = configs.make_configs("LJSpeech", scratch)
    pc = copy.deepcopy(pc)
    pc["preprocessing"]["pitch"]["feature"] = "frame_level"
    pc["preprocessing"]["energy"]["feature"] = "frame_level"
    sd = synth.fastspeech2_state_dict(pc, mc, seed=15)
    m = FastSpeech2(pc, mc); m.load_state_dict(sd); m = m.to(DEV).eval()
    spk, texts, lens, Lm = synth.make_batch(3, 40, seed=16, min_len=21)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm, p_control=1.1, pitch_level="frame_level", energy_level="frame_level")
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm, p_control=1.1)
    assert torch.equal(out[9].cpu(), ref[9]) and out[2].shape == ref[2].shape
    e = _cmp(out, ref)
    parity_log("fs2_frame_level_B3_L40", **e)
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL and max(e["pitch"], e["energy"]) < 1e-4, e


def test_fastspeech2_teacher_forced(lj_configs, parity_log):
    m, sd = _model(lj_configs, seed=5)
    spk, texts, lens, Lm = synth.make_batch(4, 48, seed=6, min_len=15)
    free = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    d_t, mel_lens = free[5].long(), free[9]
    T = int(mel_lens.max())
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm, None, mel_lens, T, free[2], free[3], d_t)
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm, None, mel_lens.to(DEV), T, free[2].to(DEV), free[3].to(DEV), d_t.to(DEV))
    e = _cmp(out, ref)
    parity_log("fs2_teacher_forced_B4_L48", **e)
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL, e
    assert torch.equal(out[9].cpu(), ref[9])


def test_fastspeech2_long_sequence_position_table(lj_configs):
    """T > max_seq_len (1000): eval mode recomputes the sinusoid table and never truncates (Models.py:145-152)."""
    pc, mc = lj_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=7, frames_per_phoneme=11.0)
    m = FastSpeech2(pc, mc); m.load_state_dict(sd); m = m.to(DEV).eval()
    spk, texts, lens, Lm = synth.make_batch(2, 120, seed=8, min_len=60)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    assert int(ref[9].max()) > 1000
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm)
    assert torch.equal(out[9].cpu(), ref[9])
    e = _cmp(out, ref)
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL, e


def test_fastspeech2_beyond_4096_frames(lj_configs, parity_log):
    """An utterance of more than 4096 mel frames (~48 s): the decoder's attention must have no length limit, as the reference has none."""
    pc, mc = lj_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=17, frames_per_phoneme=34.0)
    m = FastSpeech2(pc, mc); m.load_state_dict(sd); m = m.to(DEV).eval()
    spk, texts, lens, Lm = synth.make_batch(1, 128, seed=18)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    assert int(ref[9].max()) > 4096
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm)
    assert torch.equal(out[9].cpu(), ref[9]) and torch.equal(out[5].cpu(), ref[5])
    e = _cmp(out, ref)
    parity_log("fs2_beyond_4096_frames", **e, tmax=int(ref[9].max()))
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL, e


def test_fastspeech2_golden_vs_reference(lj_configs, libri_configs):
    """Committed outputs of the UNMODIFIED reference (tests/golden/, made by oracle/gen_golden.py)."""
    import numpy as np, os
    gdir = os.path.join(os.path.dirname(__file__), "golden")
    for name, cfgs in (("fs2_lj", lj_configs), ("fs2_libri", libri_configs)):
        z = np.load(os.path.join(gdir, name + ".npz"))
        m, sd = _model(cfgs, seed=int(z["seed"]))
        t = lambda k: torch.from_numpy(z[k])
        out = m(t("speakers").to(DEV), t("texts").to(DEV), t("src_lens").to(DEV), int(z["max_src_len"]),
                p_control=float(z["p_control"]), e_control=float(z["e_control"]), d_control=float(z["d_control"]))
        assert torch.equal(out[9].cpu(), t("mel_lens")) and torch.equal(out[5].cpu(), t("d_rounded"))
        assert (out[0].cpu() - t("mel")).abs().max() < MEL_TOL
        assert (out[1].cpu() - t("postnet_mel")).abs().max() < MEL_TOL


def _generator(seed):
    h = AttrDict(configs.HIFIGAN_CONFIG)
    sd = synth.hifigan_state_dict(h, seed=seed)
    gen = Generator(h)
    gen.load_state_dict(sd)
    gen.eval()
    gen.remove_weight_norm()
    return gen.to(DEV), sd


@pytest.mark.parametrize("B,T", [(1, 7), (2, 50), (3, 129)])
def test_hifigan_vs_oracle(B, T, parity_log):
    gen, sd = _generator(seed=1)
    mel = synth.make_mel(B, T, seed=2)
    want = O.hifigan_forward(sd, mel)
    got = gen(mel.to(DEV))
    assert got.shape == want.shape
    want64 = O.hifigan_forward(sd, mel, dtype=torch.float64)
    gen.use_tensor_cores = False; gen._invalidate()
    simt = gen(mel.to(DEV)).cpu()
    gen.use_tensor_cores = True; gen._invalidate()
    parity_log(f"hifigan_B{B}_T{T}", wav_vs_oracle32=(got.cpu() - want).abs().max(), wav_vs_oracle64=(got.cpu().double() - want64).abs().max(),
               simt_vs_oracle32=(simt - want).abs().max(), oracle32_vs_64=(want.double() - want64).abs().max(), peak=want.abs().max())
    assert (got.cpu() - want).abs().max() < WAV_TOL
    # the usual caller passes a transposed channels-last view (utils/tools.py:202)
    view = mel.transpose(1, 2).contiguous().to(DEV).transpose(1, 2)
    assert (gen(view).cpu() - want).abs().max() < WAV_TOL


@pytest.mark.parametrize("B", [16, 64])
def test_hifigan_full_size_vs_oracle(B, parity_log):
    """BASELINE.json configs[2] (B = 16) and one GPU's shard of configs[4] (B = 64): the vocoder at FULL size (x 1012 frames ->
    259072 samples per utterance).  Generator rows are independent (no cross-utterance op), so the CPU oracle is run on the first
    and last utterance of the batch and compared with those rows of the GPU result: tile indexing, the resstack slabs and the
    batch strides are exercised at the benchmarked shape while the check stays a few seconds of CPU."""
    gen, sd = _generator(seed=5)
    mel = synth.make_mel(B, 1012, seed=6)
    got = gen(mel.to(DEV))
    torch.cuda.synchronize()
    assert got.shape == (B, 1, 1012 * 256) and torch.isfinite(got).all()
    rows = [0, B - 1]
    want = O.hifigan_forward(sd, mel[rows])
    err, peak = (got[rows].cpu() - want).abs().max().item(), want.abs().max().item()
    # every other row against the same rows recomputed alone on the GPU (batch-size independence of the kernels)
    solo = gen(mel[B // 2:B // 2 + 1].to(DEV))
    err_solo = (got[B // 2:B // 2 + 1] - solo).abs().max().item()
    parity_log(f"hifigan_full_size_B{B}_T1012_vs_oracle", wav_vs_oracle32=err, peak=peak, row_alone_vs_in_batch=err_solo)
    assert err < WAV_TOL and peak > 0.3 and err_solo < 2e-6, (err, peak, err_solo)


@pytest.mark.parametrize("name", ["LJSpeech", "universal"])
def test_hifigan_real_checkpoint_vs_reference(name, parity_log):
    """The SHIPPED generator weights (hifigan/generator_*.pth.tar.zip; fixture oracle/_ref/, made by __graft_entry__.build()) through
    the reference's own call order load_state_dict -> eval -> remove_weight_norm -> to(device) (utils/model.py:62-69), against the
    unmodified reference's committed output for the same mel (tests/golden/hifigan_real_*.npz).  SURVEY.md section 7 hard part 1's worst case:
    single-pass TF32 / FP16 operands give 5e-4 here.  The shipped default policy, the all-split3 policy and the fp32 CUDA-core path
    must hold the 1e-4 bar; the all-f16+f8 policy is measured and logged only -- on the universal checkpoint it lands at 1.2e-4, which
    is why it is not the default (the truncating tensor-core accumulator, not the operand split, is the larger term: split3 6e-5)."""
    import numpy as np, os
    from oracle import real_ckpt
    sd = real_ckpt.load(name)
    if sd is None:
        pytest.skip("oracle/_ref/ real-checkpoint fixture not in this snapshot")
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"hifigan_real_{name}.npz"))
    mel, want = torch.from_numpy(z["mel"]), torch.from_numpy(z["wav"])
    gen = Generator(AttrDict(configs.HIFIGAN_CONFIG))
    gen.load_state_dict(sd)
    gen.eval()
    gen.remove_weight_norm()
    gen.to(DEV)
    errs = {}
    for label, mask in (("default", gen.f8_mask), ("split3", 0), ("f8_all_stages", 30), ("f8_all", 31)):
        gen.f8_mask = mask; gen._invalidate()
        errs[label] = (gen(mel.to(DEV)).cpu() - want).abs().max().item()
    gen.use_tensor_cores = False; gen._invalidate()
    errs["fp32_cuda_cores"] = (gen(mel.to(DEV)).cpu() - want).abs().max().item()
    parity_log(f"hifigan_real_checkpoint_{name}", **errs, peak=want.abs().max().item())
    assert max(errs[k] for k in ("default", "split3", "fp32_cuda_cores")) < WAV_TOL, errs
    assert errs["f8_all"] < 2.5e-4, errs


def test_hifigan_golden_vs_reference():
    import numpy as np, os
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "hifigan.npz"))
    gen, _ = _generator(seed=int(z["seed"]))
    got = gen(torch.from_numpy(z["mel"]).to(DEV))
    assert (got.cpu() - torch.from_numpy(z["wav"])).abs().max() < WAV_TOL


def test_end_to_end_wav(lj_configs):
    m, sd = _model(lj_configs, seed=9)
    gen, hsd = _generator(seed=3)
    spk, texts, lens, Lm = synth.make_batch(2, 32, seed=10, min_len=20)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm)
    assert torch.equal(out[9].cpu(), ref[9])
    want = O.hifigan_forward(hsd, ref[1].transpose(1, 2))
    got = gen(out[1].transpose(1, 2))
    # waveform bar applies to the vocoder given the same mel; end to end the mel error (<=1e-3) propagates, so compare both ways
    same_mel = gen(ref[1].to(DEV).transpose(1, 2))
    assert (same_mel.cpu() - want).abs().max() < WAV_TOL
    assert (got.cpu() - want).abs().max() < 5e-3


def test_synthesize_path_int16_trim_async(lj_configs, parity_log):
    """SURVEY.md section 8 f1: the sequence `synthesize.synthesize` runs per batch (synthesize.py:93-108 -> utils/tools.py:200-206 ->
    utils/model.py:74-92) with the drop-in modules and the device-side `vocoder_infer` (x32768 -> int16 + per-utterance trim fused in
    fs2_wav_to_int16, pinned async D2H): the int16 samples must equal what the reference's host-side conversion produces from the same
    fp32 waveform, every utterance trimmed to mel_len * hop."""
    from fastspeech2_b200 import dropin
    pc, mc = lj_configs
    m, sd = _model(lj_configs, seed=9)
    gen, hsd = _generator(seed=3)
    spk, texts, lens, Lm = synth.make_batch(5, 48, seed=19, min_len=20)
    batch = (["u%d" % i for i in range(5)], None, spk.numpy(), texts.numpy(), lens.numpy(), Lm)     # the 6-tuple of synthesize.py:203-210
    dev_batch = [torch.from_numpy(x).to(DEV) if hasattr(x, "dtype") else x for x in batch]          # utils.tools.to_device
    with torch.no_grad():
        out = m(*(dev_batch[2:]), p_control=1.0, e_control=1.0, d_control=1.0)
    hop = pc["preprocessing"]["stft"]["hop_length"]
    lengths = out[9] * hop
    wavs = dropin.vocoder_infer(out[1].transpose(1, 2), gen, mc, pc, lengths=lengths)
    fp32 = gen(out[1].transpose(1, 2)).squeeze(1)
    want = (fp32.cpu().numpy() * pc["preprocessing"]["audio"]["max_wav_value"]).astype("int16")     # utils/model.py:82-85
    assert len(wavs) == 5
    for i, w in enumerate(wavs):
        n = int(lengths[i])
        assert w.dtype.name == "int16" and w.shape == (n,)
        assert (w == want[i][:n]).all()
    # and against the oracle end to end (mel error <= 1e-3 propagates: a few int16 steps)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    ref_wav = O.hifigan_forward(hsd, ref[1].transpose(1, 2)).squeeze(1)
    assert torch.equal(out[9].cpu(), ref[9])
    worst = max(int(abs(w.astype("int32") - (ref_wav[i, :len(w)].numpy() * 32768).astype("int16").astype("int32")).max()) for i, w in enumerate(wavs))
    parity_log("synthesize_path_int16", worst_int16_step_vs_oracle=worst)
    assert worst <= 200          # 200 / 32768 = 6e-3: the end-to-end bound test_end_to_end_wav uses (5e-3) plus truncation


def test_batch_mode_front_end_feeds_the_gpu_path(lj_configs, parity_log, tmp_path):
    """SURVEY.md section 8 f3: `synthesize.py --mode batch` with the front-end of fastspeech2_b200/frontend.py -- a source file in the
    `val.txt` layout -> length-bucketed batches prepared in the background -> pinned staged upload -> the loop of synthesize.synthesize
    (synthesize.py:89-108: model(*(batch[2:]), controls), vocoder_infer).  Every batch is compared with the oracle run on the same
    collated (host) batch; every utterance must come back exactly once with mel_len * hop int16 samples."""
    import json
    from fastspeech2_b200 import dropin, frontend
    pc, mc = lj_configs
    m, sd = _model(lj_configs, seed=5)
    gen, hsd = _generator(seed=2)
    rng = np.random.default_rng(11)
    n_vocab = sd["encoder.src_word_emb.weight"].shape[0]
    lines = []
    for i in range(11):
        ids = rng.integers(1, n_vocab, size=int(rng.integers(9, 45)))
        lines.append(f"utt{i:02d}|LJSpeech|{{{' '.join('p%d' % v for v in ids)}}}|raw {i}")
    src = tmp_path / "val.txt"
    src.write_text("\n".join(lines) + "\n")
    pre = tmp_path / "pre"
    pre.mkdir()
    (pre / "speakers.json").write_text(json.dumps({"LJSpeech": 0}))
    fcfg = {"preprocessing": {"text": {"text_cleaners": ["english_cleaners"]}}, "path": {"preprocessed_path": str(pre)}}
    t2s = lambda text, cleaners: [int(tok[1:]) for tok in text.strip("{}").split()]
    tb = frontend.TextBatches(str(src), fcfg, batch_size=4, bucket=True, text_to_sequence=t2s, prefetch=2)
    hop = pc["preprocessing"]["stft"]["hop_length"]
    host_batches = list(tb)
    seen = []
    for k, (batch, host) in enumerate(zip(tb.device_batches(DEV), host_batches)):
        ids, raw, spk_d, texts_d, lens_d, Lm = batch
        assert ids == host[0] and spk_d.is_cuda and torch.equal(texts_d.cpu(), torch.from_numpy(host[3]))
        spk, texts, lens = (torch.from_numpy(host[i]) for i in (2, 3, 4))
        out, ref = _free_running_then_teacher_forced(m, sd, (spk, texts, lens, int(Lm)), f"batch_mode_front_end_batch{k}", parity_log)
        with torch.no_grad():
            out = m(*(batch[2:]), p_control=1.0, e_control=1.0, d_control=1.0)          # the call of synthesize.py:95-100 on the staged tensors
        wavs = dropin.vocoder_infer(out[1].transpose(1, 2), gen, mc, pc, lengths=out[9] * hop)
        assert len(wavs) == len(ids)
        for i, w in enumerate(wavs):
            assert w.dtype.name == "int16" and w.shape == (int(out[9][i]) * hop,)
        seen += ids
    assert sorted(seen) == [f"utt{i:02d}" for i in range(11)] and len(tb) == 3
