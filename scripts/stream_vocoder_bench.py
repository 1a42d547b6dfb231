"""Streamed (Generator.stream) vs offline (Generator.forward) HiFi-GAN vocoding, alternating in one process.

  shapes: configs[0] (B = 1) and configs[2] (B = 16) at 1012 mel frames, for V1 and V2, chunks of 16, 32, 64 and 128 frames.
  first_chunk_ms: host clock from the stream() call to the first chunk being complete on the device (synchronised).
  stream_ms / forward_ms: the whole batch, streamed chunk after chunk or in one forward, each ending in a device synchronise
  (median of the alternating rounds).  workspace bytes of both (fs2_vocoder_window_workspace_bytes / fs2_vocoder_workspace_bytes).
  Every streamed waveform is checked bit for bit against forward's.

Prints one JSON line per (generator, B, chunk) and a header line with the GPU name, power limit and max SM clock of this run.

usage: python scripts/stream_vocoder_bench.py [--rounds 5] [--frames 1012] [--chunks 16,32,64,128]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from fastspeech2_b200 import _lib as L, configs, synth  # noqa: E402
from fastspeech2_b200.hifigan import AttrDict, Generator  # noqa: E402


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


def generator(cfg):
    h = AttrDict(cfg)
    gen = Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=0))
    gen.eval()
    gen.remove_weight_norm()
    return gen.to("cuda")


def run_stream(gen, mel, chunk):
    """(ms to the first chunk, ms for the whole batch, the waveform)"""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    parts, first = [], None
    for _, wav in gen.stream(mel, chunk_frames=chunk):
        if first is None:
            torch.cuda.synchronize()
            first = (time.perf_counter() - t0) * 1e3
        parts.append(wav)
    torch.cuda.synchronize()
    return first, (time.perf_counter() - t0) * 1e3, torch.cat(parts, dim=2)


def run_forward(gen, mel):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    wav = gen(mel)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, wav


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=1012)
    ap.add_argument("--chunks", default="16,32,64,128")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("stream_vocoder_bench: needs a CUDA device")
    chunks = [int(c) for c in args.chunks.split(",")]
    print(json.dumps(dict(gpu_info(), frames=args.frames, rounds=args.rounds)), flush=True)
    for name, cfg in (("v1", configs.HIFIGAN_CONFIG), ("v2", configs.HIFIGAN_V2_CONFIG)):
        gen = generator(cfg)
        m = gen._pack()[0]
        for B in (1, 16):
            mel = synth.make_mel(B, args.frames, seed=1).transpose(1, 2).contiguous().to("cuda").transpose(1, 2)
            fwd_ws = L.lib().fs2_vocoder_workspace_bytes(ctypes.byref(m), B, args.frames)
            for chunk in chunks:
                run_forward(gen, mel), run_stream(gen, mel, chunk)          # warm-up: modules, workspaces, clocks
                first, total, fwd = [], [], []
                for _ in range(args.rounds):                                # alternating
                    f, t, got = run_stream(gen, mel, chunk)
                    ft, want = run_forward(gen, mel)
                    assert torch.equal(got, want), (name, B, chunk)
                    first.append(f), total.append(t), fwd.append(ft)
                print(json.dumps({
                    "generator": name, "B": B, "frames": args.frames, "chunk": chunk,
                    "first_chunk_ms": round(statistics.median(first), 3), "stream_ms": round(statistics.median(total), 3),
                    "forward_ms": round(statistics.median(fwd), 3),
                    "stream_over_forward": round(statistics.median(total) / statistics.median(fwd), 3),
                    "stream_workspace_bytes": L.lib().fs2_vocoder_window_workspace_bytes(ctypes.byref(m), B, chunk),
                    "forward_workspace_bytes": fwd_ws, "bitwise_equal": True}), flush=True)


if __name__ == "__main__":
    main()
