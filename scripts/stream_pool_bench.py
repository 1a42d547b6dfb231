"""Many live streams: the pool (one fs2_vocoder_forward_streams call per tick) against per-stream and lockstep streaming.

  workload: S streams (S = 16 and 64) of LJSpeech-like lengths (1012 +- 150 mel frames, seeded), arriving at seeded ticks over the
  first 8 ticks; V1 and V2; chunks of 32 and 64 frames.  A tick gives every live stream its next chunk.  Three arms, alternating:
    pool:     Generator.stream_pool, one call per tick;
    per_stream: one B = 1 Generator.stream per live stream per tick;
    lockstep: Generator.stream over a ragged batch of every stream that has arrived, admitting new ones only when the batch is done.
  tick_ms median / p90: host clock around one tick, ending in a device synchronise.  first_chunk_ms median / p90: from the start of a
  stream's arrival tick to the end of the tick that produced its first chunk.  samples_per_s: audio samples of all streams over the
  arm's wall time.  launches_per_tick: fs2_kernel_launch_count over the ticks.  realtime_margin: one chunk of audio at 22 050 Hz over
  the p90 tick: above 1, every live stream gets its next chunk before the previous one has played out (at this S; larger S are what
  --streams is for).
  Every stream's waveform is checked bit for bit across the arms.

Prints a header line with the GPU name, power limit and max SM clock, then one JSON line per (generator, S, chunk, arm).

usage: python scripts/stream_pool_bench.py [--rounds 3] [--streams 16,64] [--chunks 32,64] [--gens v1,v2]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from fastspeech2_b200 import _lib as L, configs, synth  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from stream_vocoder_bench import generator, gpu_info  # noqa: E402

RATE = 22050
ARMS = ("pool", "per_stream", "lockstep")


def schedule(S, seed):
    rng = np.random.default_rng(seed)
    lens = np.clip(rng.normal(1012, 150, S), 300, 1500).astype(int).tolist()
    arrive = sorted(rng.integers(0, 8, S).tolist())
    mels = [synth.make_mel(1, n, seed=seed + k)[0].to("cuda") for k, n in enumerate(lens)]
    return lens, arrive, mels


def run(arm, gen, mels, arrive, chunk, up):
    """Returns (per-tick ms, per-stream first-chunk ms, per-stream waveform, wall ms, launches)."""
    S = len(mels)
    parts = [[] for _ in range(S)]
    first = [None] * S
    tick_start = {}
    ticks = []
    pending = list(range(S))                            # not yet admitted, in arrival order
    pool = gen.stream_pool(chunk_frames=chunk) if arm == "pool" else None
    handles, iters, batch = {}, {}, None
    h = L.lib()
    torch.cuda.synchronize()
    n0, w0 = h.fs2_kernel_launch_count(), time.perf_counter()
    t = 0
    while pending or (pool is not None and len(pool)) or iters or batch is not None:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tick_start[t] = t0
        arrived = [k for k in pending if arrive[k] <= t]
        produced = []
        if arm == "pool":
            for k in arrived:
                handles[pool.add(mels[k])] = k
                pending.remove(k)
            for hd, _, wav in pool.step():
                produced.append((handles[hd], wav))
        elif arm == "per_stream":
            for k in arrived:
                iters[k] = gen.stream(mels[k][None], chunk_frames=chunk)
                pending.remove(k)
            for k in list(iters):
                try:
                    produced.append((k, next(iters[k])[1]))
                except StopIteration:
                    del iters[k]
        else:
            if batch is None and arrived:
                ks = arrived
                for k in ks:
                    pending.remove(k)
                Tm = max(mels[k].shape[1] for k in ks)
                x = torch.zeros(len(ks), 80, Tm, device="cuda")
                for i, k in enumerate(ks):
                    x[i, :, :mels[k].shape[1]] = mels[k]
                lens = torch.tensor([mels[k].shape[1] for k in ks])
                batch = (ks, gen.stream(x, mel_lens=lens, chunk_frames=chunk), 0)
            if batch is not None:
                ks, it, f0 = batch
                try:
                    _, wav = next(it)
                    for i, k in enumerate(ks):
                        n = mels[k].shape[1]
                        if f0 < n:
                            produced.append((k, wav[i:i + 1, :, :min(chunk, n - f0) * up]))
                    batch = (ks, it, f0 + chunk)
                except StopIteration:
                    batch = None
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if produced:
            ticks.append((t1 - t0) * 1e3)
        for k, wav in produced:
            if first[k] is None:
                first[k] = (t1 - tick_start[arrive[k]]) * 1e3 if arrive[k] in tick_start else (t1 - t0) * 1e3
            parts[k].append(wav)
        t += 1
    torch.cuda.synchronize()
    wall = (time.perf_counter() - w0) * 1e3
    launches = h.fs2_kernel_launch_count() - n0
    return ticks, first, [torch.cat(p, dim=2) for p in parts], wall, launches


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * len(xs)))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--streams", default="16,64")
    ap.add_argument("--chunks", default="32,64")
    ap.add_argument("--gens", default="v1,v2")
    args = ap.parse_args()
    print(json.dumps({"header": True, **gpu_info()}), flush=True)
    cfgs = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
    for g in args.gens.split(","):
        gen = generator(cfgs[g])
        up = gen._pack()[3]
        for S in [int(s) for s in args.streams.split(",")]:
            lens, arrive, mels = schedule(S, seed=100 + S)
            samples = sum(lens) * up
            for chunk in [int(c) for c in args.chunks.split(",")]:
                run("pool", gen, mels[:2], [0, 0], chunk, up)          # warm-up: kernel setup, workspaces
                res = {a: [] for a in ARMS}
                ref = None
                for _ in range(args.rounds):
                    for arm in ARMS:
                        ticks, first, wavs, wall, launches = run(arm, gen, mels, arrive, chunk, up)
                        if ref is None:
                            ref = wavs
                        assert all(torch.equal(a, b) for a, b in zip(wavs, ref)), (g, S, chunk, arm)
                        res[arm].append((ticks, first, wall, launches))
                chunk_ms = chunk * up / RATE * 1e3
                for arm in ARMS:
                    walls = [r[2] for r in res[arm]]
                    ticks = [x for r in res[arm] for x in r[0]]
                    first = [x for r in res[arm] for x in r[1]]
                    n_ticks = statistics.median(len(r[0]) for r in res[arm])
                    med = statistics.median(ticks)
                    print(json.dumps({
                        "gen": g, "S": S, "chunk_frames": chunk, "arm": arm,
                        "tick_ms_median": round(med, 3), "tick_ms_p90": round(pct(ticks, 0.9), 3),
                        "first_chunk_ms_median": round(statistics.median(first), 3), "first_chunk_ms_p90": round(pct(first, 0.9), 3),
                        "samples_per_s": round(samples / (statistics.median(walls) / 1e3)),
                        "launches_per_tick": round(statistics.median(r[3] for r in res[arm]) / n_ticks, 1),
                        "chunk_audio_ms": round(chunk_ms, 3), "realtime_margin": round(chunk_ms / pct(ticks, 0.9), 1),
                        "bit_equal_across_arms": True}), flush=True)


if __name__ == "__main__":
    main()
