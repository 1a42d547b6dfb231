"""Config dictionaries in the reference's YAML schema, plus the small JSON fixtures its constructors read.

The reference passes ``(preprocess_config, model_config)`` dicts loaded from
``config/<dataset>/{preprocess,model}.yaml`` (synthesize.py:180-185) and its constructors read
``stats.json`` / ``speakers.json`` from ``preprocess_config["path"]["preprocessed_path"]``
(model/modules.py:41-46, model/fastspeech2.py:31-37).  The GPU box has no copy of the reference tree,
so tests and bench.py build the same dict shapes here and write the two JSON files into a scratch dir.
Numeric constants are the shipped dataset statistics (preprocessed_data/*/stats.json).
"""
from __future__ import annotations

import copy
import json
import os

_STATS = {
    # [min, max, mean, std] exactly as shipped in preprocessed_data/<dataset>/stats.json
    "LJSpeech": {"pitch": [-2.917079304729967, 11.391254536985784, 207.6309860026605, 46.77559025098988],
                 "energy": [-1.431044578552246, 8.184337615966797, 37.32621679053821, 26.044180782835863]},
    "LibriTTS": {"pitch": [-2.646310080183867, 11.922013280384945, 163.55966796034886, 61.80669044989039],
                 "energy": [-1.248658537864685, 9.75546646118164, 41.65338755249414, 33.35850956918866]},
    # config/LJSpeech_paper: pitch / energy NOT normalised (preprocess.yaml:27,30), so the bin edges are raw Hz / energy.  The
    # reference ships no preprocessed_data/LJSpeech_paper/stats.json; these are representative raw LJSpeech ranges (synthetic
    # fixture values: only positivity of the pitch minimum matters for the log-spaced edges, model/modules.py:48-54).
    "LJSpeech_paper": {"pitch": [71.0, 795.8, 207.6309860026605, 46.77559025098988],
                       "energy": [0.0185, 314.96, 37.32621679053821, 26.044180782835863]},
}
_N_SPEAKERS = {"LJSpeech": 1, "LibriTTS": 904, "LJSpeech_paper": 1}

_MODEL = {
    "transformer": {"encoder_layer": 4, "encoder_head": 2, "encoder_hidden": 256,
                    "decoder_layer": 6, "decoder_head": 2, "decoder_hidden": 256,
                    "conv_filter_size": 1024, "conv_kernel_size": [9, 1],
                    "encoder_dropout": 0.2, "decoder_dropout": 0.2},
    "variance_predictor": {"filter_size": 256, "kernel_size": 3, "dropout": 0.5},
    "variance_embedding": {"pitch_quantization": "linear", "energy_quantization": "linear", "n_bins": 256},
    "multi_speaker": False,
    "max_seq_len": 1000,
    "vocoder": {"model": "HiFi-GAN", "speaker": "LJSpeech"},
}

HIFIGAN_CONFIG = {
    "resblock": "1", "upsample_rates": [8, 8, 2, 2], "upsample_kernel_sizes": [16, 16, 4, 4],
    "upsample_initial_channel": 512, "resblock_kernel_sizes": [3, 7, 11],
    "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
    "num_mels": 80, "hop_size": 256, "sampling_rate": 22050,
}

# HiFi-GAN V2: V1 with upsample_initial_channel 128, so its stages are 64, 32, 16 and 8 channels wide (0.93 M parameters)
HIFIGAN_V2_CONFIG = dict(HIFIGAN_CONFIG, upsample_initial_channel=128)


def make_configs(dataset: str, scratch_dir: str):
    """Return (preprocess_config, model_config) and materialise stats.json / speakers.json."""
    if dataset not in _STATS:
        raise ValueError(f"unknown dataset {dataset!r}")
    path = os.path.join(scratch_dir, "preprocessed_data", dataset)
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "stats.json"), "w") as f:
        json.dump(_STATS[dataset], f)
    n_spk = _N_SPEAKERS[dataset]
    with open(os.path.join(path, "speakers.json"), "w") as f:
        json.dump({f"spk{i}": i for i in range(n_spk)} if n_spk > 1 else {dataset: 0}, f)
    preprocess = {
        "dataset": dataset,
        "path": {"preprocessed_path": path},
        "preprocessing": {
            "audio": {"sampling_rate": 22050, "max_wav_value": 32768.0},
            "stft": {"filter_length": 1024, "hop_length": 256, "win_length": 1024},
            "mel": {"n_mel_channels": 80, "mel_fmin": 0, "mel_fmax": 8000},
            "pitch": {"feature": "phoneme_level", "normalization": True},
            "energy": {"feature": "phoneme_level", "normalization": True},
        },
    }
    model = copy.deepcopy(_MODEL)
    model["multi_speaker"] = n_spk > 1
    if dataset == "LibriTTS":
        model["vocoder"]["speaker"] = "universal"
    if dataset == "LJSpeech_paper":                    # config/LJSpeech_paper/{model,preprocess}.yaml
        model["transformer"]["decoder_layer"] = 4
        model["variance_embedding"]["pitch_quantization"] = "log"
        for k in ("pitch", "energy"):
            preprocess["preprocessing"][k] = {"feature": "frame_level", "normalization": False}
    return preprocess, model
