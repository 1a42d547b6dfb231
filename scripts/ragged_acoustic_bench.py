"""Padded vs ragged FastSpeech2 (forward(ragged=False / True)), alone and followed by the HiFi-GAN vocoder (padded: Generator(mel);
ragged: Generator(mel, mel_lens)), alternating in one process, CUDA-event timed.

  configs[3]: the LibriTTS batch bench.py builds (make_batch(64, 256, seed=11, n_speakers=904, min_len=64)), free-running.

Prints one JSON line: the GPU name, power limit and max SM clock queried in the same run; valid / padded frames; the work the ragged
mode skips, counted from the lengths (decoder attention 128 x 128 tile pairs sum_b ceil(n_b/128)^2 against B * ceil(T/128)^2,
128-row conv tiles of the encoder and the decoder); ms per call of each mode (median of the alternating rounds) and valid mel frames
per second.

usage: python scripts/ragged_acoustic_bench.py [--rounds 5] [--calls 10] [--warmup-s 1.0]
"""
import argparse
import contextlib
import io
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

from fastspeech2_b200 import configs, synth  # noqa: E402
from fastspeech2_b200.hifigan import AttrDict, Generator  # noqa: E402
from fastspeech2_b200.model import FastSpeech2  # noqa: E402
from ragged_vocoder_bench import gpu_info, time_calls  # noqa: E402


def tiles(lens, T, tile=128):
    live = sum(-(-int(n) // tile) for n in lens)
    return {"live": live, "padded": len(lens) * -(-T // tile)}


def attention_pairs(lens, T, tile=128):
    return {"live": sum((-(-int(n) // tile)) ** 2 for n in lens), "padded": len(lens) * (-(-T // tile)) ** 2}


def compare(modes, rounds, calls, warmup_s):
    t_end = time.perf_counter() + warmup_s
    while time.perf_counter() < t_end:               # clocks and caches settle; both modes' workspaces are allocated
        for fn in modes.values():
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in modes}
    for _ in range(rounds):
        for k, fn in modes.items():                  # alternating: slow drifts of the clock hit both modes alike
            ms[k].append(time_calls(fn, calls))
    med = {k: statistics.median(v) for k, v in ms.items()}
    return {"padded_ms": round(med["padded"], 3), "ragged_ms": round(med["ragged"], 3),
            "ragged_over_padded": round(med["ragged"] / med["padded"], 4),
            "padded_ms_rounds": [round(v, 3) for v in ms["padded"]], "ragged_ms_rounds": [round(v, 3) for v in ms["ragged"]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup-s", type=float, default=1.0)
    args = ap.parse_args()
    dev = torch.device("cuda")
    pc, mc = configs.make_configs("LibriTTS", tempfile.mkdtemp())
    model = FastSpeech2(pc, mc)
    model.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=0))
    model = model.to(dev).eval()
    voc = Generator(AttrDict(configs.HIFIGAN_CONFIG))
    voc.load_state_dict(synth.hifigan_state_dict(configs.HIFIGAN_CONFIG, seed=0))
    voc.eval()
    with contextlib.redirect_stdout(io.StringIO()):
        voc.remove_weight_norm()
    voc.to(dev)
    batch = [t.to(dev) if torch.is_tensor(t) else t for t in synth.make_batch(64, 256, seed=11, n_speakers=904, min_len=64)]
    spk, texts, lens, L = batch
    with torch.no_grad():
        pad = model(*batch, ragged=False)
        rag = model(*batch, ragged=True)
    mel_lens = rag[9].cpu().tolist()
    T = int(rag[0].shape[1])
    valid = sum(mel_lens)

    def fs2(ragged):
        return lambda: model(*batch, ragged=ragged)

    def chain(ragged):
        def run():
            out = model(*batch, ragged=ragged)
            return voc(out[1].transpose(1, 2), mel_lens=out[9]) if ragged else voc(out[1].transpose(1, 2))
        return run

    res = {"bench": "ragged_acoustic", **gpu_info(), "config": "configs[3] LibriTTS B=64 make_batch(64, 256, seed=11, min_len=64)",
           "B": len(mel_lens), "T": T, "valid_frames": valid, "padded_frames": len(mel_lens) * T,
           "same_mel_lens": bool(torch.equal(pad[9], rag[9])),
           "work": {"decoder_attention_tile_pairs": attention_pairs(mel_lens, T), "decoder_conv_row_tiles": tiles(mel_lens, T),
                    "encoder_conv_row_tiles": tiles(lens.cpu().tolist(), int(L))}}
    with torch.no_grad():
        r = compare({"padded": fs2(False), "ragged": fs2(True)}, args.rounds, args.calls, args.warmup_s)
        r.update({f"valid_frames_per_s_{k}": round(valid / (r[f"{k}_ms"] / 1e3)) for k in ("padded", "ragged")})
        res["fastspeech2"] = r
        r = compare({"padded": chain(False), "ragged": chain(True)}, args.rounds, max(1, args.calls // 5), args.warmup_s)
        r.update({f"valid_frames_per_s_{k}": round(valid / (r[f"{k}_ms"] / 1e3)) for k in ("padded", "ragged")})
        res["fastspeech2_and_vocoder"] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
