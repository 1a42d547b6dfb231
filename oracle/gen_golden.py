"""Generate tests/golden/* by running the UNMODIFIED reference (imported read-only from /root/reference) on CPU.

Run once in the build container:  python -m oracle.gen_golden
The fixtures hold inputs and the reference's OUTPUTS only; weights are regenerated from the seed by
fastspeech2_b200.synth (a pure function of the spec and seed), loaded into the reference with load_state_dict(strict).
The reference ships no golden vectors of its own (SURVEY.md section 4), so these files are the pin.
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastspeech2_b200 import configs, synth  # noqa: E402
from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def paper_state_dict(pc, mc, seed):
    """LJSpeech_paper weights: the unnormalised pitch / energy predictors are steered into their (raw-valued) bin ranges so that the
    log-spaced pitch edges and many distinct buckets are exercised."""
    sd = synth.fastspeech2_state_dict(pc, mc, seed=seed)
    sd["variance_adaptor.pitch_predictor.linear_layer.bias"].fill_(220.0)
    sd["variance_adaptor.pitch_predictor.linear_layer.weight"] *= 250
    sd["variance_adaptor.energy_predictor.linear_layer.bias"].fill_(60.0)
    sd["variance_adaptor.energy_predictor.linear_layer.weight"] *= 100
    return sd


def main():
    torch.set_num_threads(1)      # pin the thread count: run-to-run bitwise reproducible (SURVEY.md Appendix D)
    FastSpeech2, hifigan = ref_import.load()
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp()
    keys = {}
    cases = [("fs2_lj", "LJSpeech", 11, dict(batch=2, max_len=24, seed=21, min_len=15), dict(p_control=1.0, e_control=1.0, d_control=1.0)),
             ("fs2_libri", "LibriTTS", 12, dict(batch=3, max_len=32, seed=22, min_len=12, n_speakers=904),
              dict(p_control=1.1, e_control=0.9, d_control=0.8))]
    for name, ds, seed, bk, ctl in cases:
        pc, mc = configs.make_configs(ds, tmp)
        sd = synth.fastspeech2_state_dict(pc, mc, seed=seed)
        ref = FastSpeech2(pc, mc)
        ref.load_state_dict(sd, strict=True)
        ref.eval()
        keys[ds] = {k: list(v.shape) for k, v in ref.state_dict().items()}
        spk, texts, lens, L = synth.make_batch(**bk)
        with torch.no_grad():
            out = ref(spk, texts, lens, L, **ctl)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), seed=seed, speakers=spk.numpy(), texts=texts.numpy(),
                            src_lens=lens.numpy(), max_src_len=L, mel=out[0].numpy(), postnet_mel=out[1].numpy(),
                            p_pred=out[2].numpy(), e_pred=out[3].numpy(), logd=out[4].numpy(), d_rounded=out[5].numpy(),
                            src_masks=out[6].numpy(), mel_masks=out[7].numpy(), mel_lens=out[9].numpy(), **ctl)
        print(name, "mel", tuple(out[0].shape), "mel_lens", out[9].tolist())

    h = hifigan.AttrDict(configs.HIFIGAN_CONFIG)
    seed = 13
    hsd = synth.hifigan_state_dict(h, seed=seed)
    gen = hifigan.Generator(h)
    gen.load_state_dict(hsd, strict=True)
    keys["hifigan_weight_norm"] = {k: list(v.shape) for k, v in gen.state_dict().items()}
    gen.eval()
    gen.remove_weight_norm()
    keys["hifigan_folded"] = {k: list(v.shape) for k, v in gen.state_dict().items()}
    mel = synth.make_mel(2, 24, seed=23)
    with torch.no_grad():
        wav = gen(mel)
    np.savez_compressed(os.path.join(OUT, "hifigan.npz"), seed=seed, mel=mel.numpy(), wav=wav.numpy())
    print("hifigan wav", tuple(wav.shape), "peak", float(wav.abs().max()))
    # config/LJSpeech_paper: 4-layer decoder, frame-level unnormalised pitch / energy, log-spaced pitch edges (SURVEY.md section 8 f2)
    pc, mc = configs.make_configs("LJSpeech_paper", tmp)
    seed = 14
    sd = paper_state_dict(pc, mc, seed)
    ref = FastSpeech2(pc, mc)
    ref.load_state_dict(sd, strict=True)
    ref.eval()
    keys["LJSpeech_paper"] = {k: list(v.shape) for k, v in ref.state_dict().items()}
    spk, texts, lens, L = synth.make_batch(batch=3, max_len=30, seed=24, min_len=14)
    with torch.no_grad():
        out = ref(spk, texts, lens, L, p_control=1.05)
    np.savez_compressed(os.path.join(OUT, "fs2_lj_paper.npz"), seed=seed, speakers=spk.numpy(), texts=texts.numpy(),
                        src_lens=lens.numpy(), max_src_len=L, mel=out[0].numpy(), postnet_mel=out[1].numpy(),
                        p_pred=out[2].numpy(), e_pred=out[3].numpy(), logd=out[4].numpy(), d_rounded=out[5].numpy(),
                        src_masks=out[6].numpy(), mel_masks=out[7].numpy(), mel_lens=out[9].numpy(), p_control=1.05, e_control=1.0, d_control=1.0)
    nb = torch.bucketize(out[2], sd["variance_adaptor.pitch_bins"]).unique().numel()
    print("fs2_lj_paper mel", tuple(out[0].shape), "mel_lens", out[9].tolist(), "distinct log-spaced pitch buckets", nb)

    # the shipped generator checkpoints (real weights): outputs of the unmodified reference Generator on a synthetic mel
    from oracle import real_ckpt
    for name in ("LJSpeech", "universal"):
        gen = hifigan.Generator(h)
        gen.load_state_dict(real_ckpt.read_reference_checkpoint(name), strict=True)     # utils/model.py:62-66
        gen.eval()
        gen.remove_weight_norm()
        mel = synth.make_mel(2, 96, seed=25)
        with torch.no_grad():
            wav = gen(mel)
        np.savez_compressed(os.path.join(OUT, f"hifigan_real_{name}.npz"), mel=mel.numpy(), wav=wav.numpy())
        print("hifigan real", name, tuple(wav.shape), "peak", float(wav.abs().max()))
    with open(os.path.join(OUT, "state_dict_keys.json"), "w") as f:
        json.dump(keys, f, indent=0, sort_keys=True)


def live_cases():
    """tests/golden/reference_cases.npz: the reference's outputs for the inputs of test_oracle_golden.py's multi-speaker / teacher-forced /
    vocoder case and its frame-level case (inputs are regenerated from the same seeds by the tests)."""
    import copy
    FastSpeech2, hifigan = ref_import.load()
    scratch = tempfile.mkdtemp()
    z = {}
    pc, mc = configs.make_configs("LibriTTS", scratch)
    sd = synth.fastspeech2_state_dict(pc, mc, seed=31)
    ref = FastSpeech2(pc, mc)
    ref.load_state_dict(sd, strict=True)
    ref.eval()
    spk, texts, lens, L = synth.make_batch(3, 36, seed=32, n_speakers=904, min_len=10)
    with torch.no_grad():
        want = ref(spk, texts, lens, L, p_control=0.9, d_control=1.2)
        ml = want[9]
        want2 = ref(spk, texts, lens, L, None, ml, int(ml.max()), want[2], want[3], want[5].long())
    for i in (0, 1, 2, 3, 4, 5, 9):
        z[f"free_{i}"] = want[i].numpy()
    for i in (0, 1, 4):      # fed its own predictions, the teacher-forced mel and log-durations equal the free-running ones bit for bit
        assert torch.equal(want2[i], want[i])
    for i in (2, 3):
        z[f"forced_{i}"] = want2[i].numpy()
    h = hifigan.AttrDict(configs.HIFIGAN_CONFIG)
    gen = hifigan.Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=33), strict=True)
    gen.eval()
    gen.remove_weight_norm()
    with torch.no_grad():
        z["wav"] = gen(synth.make_mel(1, 30, seed=34)).numpy()
    pc, mc = configs.make_configs("LJSpeech", scratch)
    pc = copy.deepcopy(pc)
    pc["preprocessing"]["pitch"]["feature"] = "frame_level"
    pc["preprocessing"]["energy"]["feature"] = "frame_level"
    ref = FastSpeech2(pc, mc)
    ref.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=41), strict=True)
    ref.eval()
    spk, texts, lens, L = synth.make_batch(2, 22, seed=42, min_len=13)
    with torch.no_grad():
        want = ref(spk, texts, lens, L, p_control=1.2)
    for i in (0, 1, 2, 3, 4, 9):
        z[f"frame_{i}"] = want[i].numpy()
    np.savez_compressed(os.path.join(OUT, "reference_cases.npz"), **z)


def frontend_cases():
    """tests/golden/frontend_reference_batches.npz: the three `preprocessed_data/*/val.txt` files the reference ships, the token
    sequences its `text_to_sequence` makes of every line, and the batches of its TextDataset + DataLoader(batch_size=8).  Runs the
    reference's modules (`text`, `dataset`) from its own tree, so call it in a process of its own."""
    ref_import._stub()
    ref = ref_import.REFERENCE_ROOT
    sys.path.insert(0, ref)
    os.chdir(ref)
    import yaml
    from torch.utils.data import DataLoader
    from dataset import TextDataset as RefTextDataset
    from text import text_to_sequence
    z = {}
    as_bytes = lambda s: np.frombuffer(s.encode("utf-8") if isinstance(s, str) else s, dtype=np.uint8)
    for ds in ("LJSpeech", "LibriTTS", "AISHELL3"):
        pc = yaml.safe_load(open(f"config/{ds}/preprocess.yaml"))
        pre = pc["path"]["preprocessed_path"]
        src = os.path.join(pre, "val.txt")
        cleaners = pc["preprocessing"]["text"]["text_cleaners"]
        data = RefTextDataset(src, pc)
        seqs = [np.asarray(text_to_sequence(t, cleaners), dtype=np.int64) for t in data.text]
        z[f"{ds}__val"] = as_bytes(open(src, "rb").read())
        z[f"{ds}__speakers"] = as_bytes(open(os.path.join(pre, "speakers.json"), "rb").read())
        z[f"{ds}__seq"] = np.concatenate(seqs)
        z[f"{ds}__seq_len"] = np.array([len(s) for s in seqs], dtype=np.int64)
        meta = {"cleaners": cleaners, "batches": [], "item5": None}
        for i, (ids, raws, spk, texts, lens, mx) in enumerate(DataLoader(data, batch_size=8, collate_fn=data.collate_fn)):
            meta["batches"].append({"ids": ids, "raw": raws, "max": int(mx), "max_type": type(mx).__name__})
            z[f"{ds}__b{i}__spk"], z[f"{ds}__b{i}__texts"], z[f"{ds}__b{i}__lens"] = spk, texts, lens
        it = data[5]
        assert np.array_equal(it[2], seqs[5])
        meta["item5"] = [it[0], int(it[1]), it[3]]
        z[f"{ds}__meta"] = as_bytes(json.dumps(meta))
    np.savez_compressed(os.path.join(OUT, "frontend_reference_batches.npz"), **z)


if __name__ == "__main__":
    if "--frontend" in sys.argv:
        frontend_cases()
    elif "--cases" in sys.argv:
        live_cases()
    else:
        main()
