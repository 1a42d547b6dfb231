"""Padded vs ragged HiFi-GAN vocoding (Generator.forward without / with mel_lens), alternating in one process, CUDA-event timed.

  configs[3]: the LibriTTS batch bench.py builds (make_batch(64, 256, seed=11, n_speakers=904, min_len=64)) run free through FastSpeech2;
              the vocoder gets out[1] padded (mel_lens=None) or ragged (mel_lens=out[9]): the work on padded frames is what ragged skips.
  configs[2]: B = 16 x 1012 frames with every length equal to T: nothing can be skipped, so this is the ragged path's overhead.

Prints one JSON line: valid / padded frames, ms per call of each mode (median of the alternating rounds), valid audio samples per
second, and the GPU name, power limit and max SM clock queried in the same run.

usage: python scripts/ragged_vocoder_bench.py [--rounds 5] [--calls 10] [--warmup-s 1.0]
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from fastspeech2_b200 import configs, synth  # noqa: E402
from fastspeech2_b200.hifigan import AttrDict, Generator  # noqa: E402
from fastspeech2_b200.model import FastSpeech2  # noqa: E402


def gpu_info():
    """name, power limit and max SM clock of the visible GPU (query only)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        dev = torch.cuda.current_device()
        name, power, clock = [s.strip() for s in out[min(dev, len(out) - 1)].split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:       # report, never fail the measurement over it
        return {"gpu": torch.cuda.get_device_name(), "power_limit": f"unavailable ({type(e).__name__})"}


def time_calls(fn, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(calls):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def compare(voc, mel, mel_lens, rounds, calls, warmup_s):
    modes = {"padded": lambda: voc(mel), "ragged": lambda: voc(mel, mel_lens=mel_lens)}
    t_end = time.perf_counter() + warmup_s
    while time.perf_counter() < t_end:               # clocks and caches settle; both modes' workspaces are allocated
        for fn in modes.values():
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in modes}
    for _ in range(rounds):
        for k, fn in modes.items():                  # alternating: slow drifts of the clock hit both modes alike
            ms[k].append(time_calls(fn, calls))
    valid = int(mel_lens.sum().item())
    B, _, T = mel.shape
    med = {k: statistics.median(v) for k, v in ms.items()}
    return {"B": B, "T": T, "valid_frames": valid, "padded_frames": B * T,
            "padded_ms": round(med["padded"], 3), "ragged_ms": round(med["ragged"], 3),
            "ragged_over_padded": round(med["ragged"] / med["padded"], 4),
            "padded_ms_rounds": [round(v, 3) for v in ms["padded"]], "ragged_ms_rounds": [round(v, 3) for v in ms["ragged"]],
            "valid_samples_per_s_padded": round(valid * 256 / (med["padded"] / 1e3)),
            "valid_samples_per_s_ragged": round(valid * 256 / (med["ragged"] / 1e3))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup-s", type=float, default=1.0)
    args = ap.parse_args()
    dev = torch.device("cuda")
    voc = Generator(AttrDict(configs.HIFIGAN_CONFIG))
    voc.load_state_dict(synth.hifigan_state_dict(configs.HIFIGAN_CONFIG, seed=0))
    voc.eval()
    with contextlib.redirect_stdout(io.StringIO()):
        voc.remove_weight_norm()
    voc.to(dev)
    pc, mc = configs.make_configs("LibriTTS", tempfile.mkdtemp())
    model = FastSpeech2(pc, mc)
    model.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=0))
    model = model.to(dev).eval()
    spk, texts, lens, L = synth.make_batch(64, 256, seed=11, n_speakers=904, min_len=64)
    with torch.no_grad():
        out = model(spk.to(dev), texts.to(dev), lens.to(dev), L)
    res = {"bench": "ragged_vocoder", **gpu_info()}
    res["configs3"] = compare(voc, out[1].transpose(1, 2), out[9], args.rounds, args.calls, args.warmup_s)
    del model, out
    mel = synth.make_mel(16, 1012, seed=0).to(dev)
    res["configs2_all_full"] = compare(voc, mel, torch.full((16,), 1012, dtype=torch.int32, device=dev), args.rounds, args.calls,
                                       args.warmup_s)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
