"""Sample-rate conversion on the GPU: the resampler kernel against its HBM bound and against the vocoder, and its cost in a stream pool.

  kernel: Resampler(22050, R) on configs[2]'s waveform (B = 16 x 1012 mel frames = 259 072 samples per row, V1 generator output),
    CUDA events around `--iters` launches after a warm-up.  The kernel must read every input sample and write every output sample once:
    bytes = 4 B N + 4 B ceil(N R / 22050) (fp32 in and out); hbm_bound_us = bytes / 3.35 TB/s (the H100 SXM data sheet; not a measured
    peak), so share_of_hbm_bound = hbm_bound_us / kernel_us.  The vocoder's Generator.forward on the same mel is timed the same way.
  pool: scripts/stream_pool_bench.py's workload (S = 16 streams of 1012 +- 150 frames arriving over the first 8 ticks, V1, chunks of
    64 frames), median host-clock tick (ending in a device synchronise) of Generator.stream_pool with sample_rate None and each R,
    alternating the arms over `--rounds` rounds.

Prints a header line with the GPU name, power limit and max SM clock, then one JSON line per measurement.

usage: python scripts/resample_bench.py [--iters 50] [--rounds 3] [--rates 16000,48000,24000,44100,8000]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import torch  # noqa: E402

from fastspeech2_b200 import configs, synth  # noqa: E402
from fastspeech2_b200.resample import Resampler  # noqa: E402
from stream_pool_bench import schedule  # noqa: E402
from stream_vocoder_bench import generator, gpu_info  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def event_ms(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def pool_ticks(gen, mels, arrive, chunk, rate):
    pool = gen.stream_pool(chunk_frames=chunk, sample_rate=rate)
    pending, ticks, t = list(range(len(mels))), [], 0
    while pending or len(pool):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in [k for k in pending if arrive[k] <= t]:
            pool.add(mels[k])
            pending.remove(k)
        pool.step()
        torch.cuda.synchronize()
        ticks.append((time.perf_counter() - t0) * 1e3)
        t += 1
    return ticks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rates", default="16000,48000,24000,44100,8000")
    args = ap.parse_args()
    rates = [int(r) for r in args.rates.split(",")]
    print(json.dumps(gpu_info()))
    gen = generator(configs.HIFIGAN_CONFIG)
    mel = synth.make_mel(16, 1012, seed=0).to("cuda")
    voc_ms = event_ms(lambda: gen(mel), max(3, args.iters // 10))
    print(json.dumps({"what": "vocoder_forward", "B": 16, "frames": 1012, "ms": round(voc_ms, 3)}))
    wav = gen(mel)
    B, N = wav.shape[0], wav.shape[2]
    for rate in rates:
        rs = Resampler(22050, rate)
        n_out = rs.n_out(N)
        us = event_ms(lambda: rs(wav), args.iters) * 1e3
        byts = 4 * B * (N + n_out)
        bound = byts / HBM_BYTES_PER_S * 1e6
        print(json.dumps({"what": "resample_kernel", "rate": rate, "up": rs.up, "down": rs.down, "K": rs.K, "B": B, "N": N,
                          "n_out": n_out, "bytes": byts, "kernel_us": round(us, 2), "hbm_bound_us": round(bound, 2),
                          "share_of_hbm_bound": round(bound / us, 3), "share_of_vocoder_forward": round(us / 1e3 / voc_ms, 5)}))
    _lens, arrive, mels = schedule(16, seed=0)
    arms = [None] + rates
    ticks = {a: [] for a in arms}
    for _ in range(args.rounds):
        for a in arms:
            ticks[a] += pool_ticks(gen, mels, arrive, 64, a)
    for a in arms:
        print(json.dumps({"what": "stream_pool_tick", "S": 16, "chunk": 64, "sample_rate": a,
                          "tick_ms_median": round(statistics.median(ticks[a]), 3), "ticks": len(ticks[a])}))


if __name__ == "__main__":
    main()
