"""Generate tests/golden/fs2_controls.npz by running the UNMODIFIED reference (imported read-only) on CPU, one thread, with tensor
p / e / d controls: per utterance ([B, 1]) and per phoneme ([B, L]), broadcast by the reference's `prediction * control`
(model/modules.py:85,96,132-135).

Run once in the build container:  python -m oracle.gen_golden_controls
Case <c> is stored under keys "<c>__<name>": its dataset, weight seed, inputs, controls and the reference's 10-tuple.  Weights are
regenerated from the seed by fastspeech2_b200.synth (LJSpeech_paper: gen_golden.paper_state_dict), as for the other fixtures.
"""
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastspeech2_b200 import configs, synth  # noqa: E402
from oracle import ref_import  # noqa: E402
from oracle.gen_golden import paper_state_dict  # noqa: E402

OUTPUTS = ("mel", "postnet_mel", "p_pred", "e_pred", "logd", "d_rounded", "src_masks", "mel_masks", "src_lens_out", "mel_lens")


def controls(B, L, seed, p_cols, d_cols):
    """p in [0.8, 1.25], d in [0.5, 2]: [B, cols] with cols 1 (per utterance) or L (per phoneme)."""
    g = torch.Generator().manual_seed(seed)
    p = 0.8 + 0.45 * torch.rand(B, L if p_cols == "L" else 1, generator=g)
    d = 0.5 + 1.5 * torch.rand(B, L if d_cols == "L" else 1, generator=g)
    return p, d


# name: (dataset, weight seed, make_batch kwargs, p columns, d columns, e_control)
CASES = {
    "lj_utt": ("LJSpeech", 61, dict(batch=2, max_len=18, seed=62, min_len=12), "1", "1", None),
    "lj_phoneme": ("LJSpeech", 63, dict(batch=2, max_len=18, seed=64, min_len=12), "L", "L", None),
    # e_control is never read by the reference (modules.py:124): a tensor that broadcasts to nothing
    "libri_utt": ("LibriTTS", 65, dict(batch=2, max_len=20, seed=66, min_len=12, n_speakers=904), "1", "1", "tensor"),
    "paper_utt_phoneme": ("LJSpeech_paper", 67, dict(batch=2, max_len=18, seed=68, min_len=12), "1", "L", None),
}


def main():
    torch.set_num_threads(1)      # run-to-run bitwise reproducible, as gen_golden
    FastSpeech2, _ = ref_import.load()
    tmp = tempfile.mkdtemp()
    z = {}
    for name, (ds, seed, bk, p_cols, d_cols, e_kind) in CASES.items():
        pc, mc = configs.make_configs(ds, tmp)
        sd = paper_state_dict(pc, mc, seed) if ds == "LJSpeech_paper" else synth.fastspeech2_state_dict(pc, mc, seed=seed)
        ref = FastSpeech2(pc, mc)
        ref.load_state_dict(sd, strict=True)
        ref.eval()
        spk, texts, lens, L = synth.make_batch(**bk)
        p, d = controls(len(lens), L, seed + 100, p_cols, d_cols)
        e = torch.full((7,), 0.5) if e_kind == "tensor" else 1.0
        with torch.no_grad():
            out = ref(spk, texts, lens, L, p_control=p, e_control=e, d_control=d)
        rec = dict(dataset=np.array(ds), seed=seed, speakers=spk.numpy(), texts=texts.numpy(), src_lens=lens.numpy(), max_src_len=L,
                   p_control=p.numpy(), d_control=d.numpy(), e_control=np.asarray(e))
        rec.update({k: v.numpy() for k, v in zip(OUTPUTS, out)})
        z.update({f"{name}__{k}": v for k, v in rec.items()})
        print(name, ds, "mel", tuple(out[0].shape), "mel_lens", out[9].tolist())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "fs2_controls.npz"), **z)


if __name__ == "__main__":
    main()
