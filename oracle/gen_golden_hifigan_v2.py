"""Generate tests/golden/hifigan_v2.npz by running the UNMODIFIED reference HiFi-GAN Generator (imported read-only) on CPU, one thread,
with the V2 config (configs.HIFIGAN_V2_CONFIG: upsample_initial_channel 128, so stages of 64, 32, 16 and 8 channels).

Run once in the build container:  python -m oracle.gen_golden_hifigan_v2
Stores the weight seed, the mel batch (synth.make_mel) and the reference's waveform, and the reference's state_dict key -> shape maps in
the checkpoint (weight-norm) layout and after remove_weight_norm (folded), as JSON strings.  Weights are regenerated from the seed by
fastspeech2_b200.synth.hifigan_state_dict, as for the other fixtures.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastspeech2_b200 import configs, synth  # noqa: E402
from oracle import ref_import  # noqa: E402

SEED = 71
MEL = dict(batch=2, frames=29, seed=72)


def main():
    torch.set_num_threads(1)      # run-to-run bitwise reproducible, as gen_golden
    _, hifigan = ref_import.load()
    h = hifigan.AttrDict(configs.HIFIGAN_V2_CONFIG)
    gen = hifigan.Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=SEED), strict=True)
    keys_wn = {k: list(v.shape) for k, v in gen.state_dict().items()}
    gen.eval()
    gen.remove_weight_norm()
    keys_folded = {k: list(v.shape) for k, v in gen.state_dict().items()}
    mel = synth.make_mel(**MEL)
    with torch.no_grad():
        wav = gen(mel)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "hifigan_v2.npz"), seed=SEED, mel=mel.numpy(), wav=wav.numpy(),
                        keys_weight_norm=np.array(json.dumps(keys_wn)), keys_folded=np.array(json.dumps(keys_folded)))
    print("hifigan V2 wav", tuple(wav.shape), "peak", float(wav.abs().max()), "keys", len(keys_wn), len(keys_folded))


if __name__ == "__main__":
    main()
