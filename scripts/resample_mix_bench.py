"""Many output formats in one stream pool: one pool whose streams each have their own rate and encoding (StreamPool.add(mel,
sample_rate, encoding), one fs2_resample_streams_mixed launch per tick) against one single-format pool per format.

  workload: scripts/stream_pool_bench.py's traffic -- S = 64 streams of LJSpeech-like lengths (1012 +- 150 mel frames, seeded) arriving
  at seeded ticks over the first 8 ticks, 32-frame chunks, V1 and V2 -- with the streams spread evenly over four formats a TTS server
  meets: 8 kHz G.711 mu-law (telephony), 16 kHz int16 PCM (speech recognition), 24 kHz fp32 and 48 kHz int16 PCM (web and apps).
  Two arms, alternating over `--rounds` rounds:
    mixed: one Generator.stream_pool; every stream added with its format;
    split: four Generator.stream_pool(sample_rate=R), one per format, all stepped in each tick.
  tick_ms median / p90: host clock around one tick, ending in a device synchronise.  first_chunk_ms median / p90: from the start of a
  stream's arrival tick to the end of the tick that produced its first chunk.  launches_per_tick: fs2_kernel_launch_count over the
  ticks.  d2h_bytes_per_tick: the bytes of the tick's chunks, what a device-to-host copy of the outputs would move.
  conversion (mixed arm): CUDA events around each tick's conversion call (its record upload and the kernel); bytes = 4 x the input
  span its outputs read + the output bytes, per stream; hbm_bound_us = bytes / 3.35 TB/s (the H100 SXM data sheet, not a measured
  peak); share_of_hbm_bound = hbm_bound_us / the call's time.  Medians over the ticks.
  Every stream's output is checked bit for bit across the arms.

Prints a header line with the GPU name, power limit and max SM clock, then one JSON line per (generator, arm).

usage: python scripts/resample_mix_bench.py [--rounds 3] [--streams 64] [--chunk 32] [--gens v1,v2]
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

from fastspeech2_b200 import _lib as L, configs  # noqa: E402
from stream_pool_bench import pct, schedule  # noqa: E402
from stream_vocoder_bench import generator, gpu_info  # noqa: E402

FORMATS = ((8000, "ulaw"), (16000, "pcm16"), (24000, "f32"), (48000, "pcm16"))
HBM_BYTES_PER_S = 3.35e12
ARMS = ("mixed", "split")


def conversion_bytes(records):
    """Bytes a conversion call must move: each stream's input span (fp32) and its outputs."""
    total = 0
    for x0, x1, i0, i1, i2, n, j0, j1, rs, enc in records:
        if j1 <= j0:
            continue
        if rs.identity:
            lo, hi = j0, min(j1, n)
        else:
            lo = max((j0 * rs.down + rs.half_len) // rs.up - rs.K + 1, 0)
            hi = min(((j1 - 1) * rs.down + rs.half_len) // rs.up + 1, n)
        total += 4 * max(hi - lo, 0) + (j1 - j0) * (4 if enc == L.RESAMPLE_F32 else 2 if enc == L.RESAMPLE_PCM16 else 1)
    return total


def timed(pool, log):
    """Wraps the pool's conversion call in CUDA events; log gets (start, end, bytes) per call."""
    inner = pool._resample

    def call(records, max_out):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = inner(records, max_out)
        b.record()
        log.append((a, b, conversion_bytes(records)))
        return out
    call.rs = inner.rs
    pool._resample = call


def run(arm, gen, mels, arrive, chunk, log=None):
    """Returns (per-tick ms, per-stream first-chunk ms, per-stream output, launches, D2H bytes)."""
    S = len(mels)
    fmt = [FORMATS[k % len(FORMATS)] for k in range(S)]
    if arm == "mixed":
        pools = [gen.stream_pool(chunk_frames=chunk)]
        if log is not None:
            timed(pools[0], log)
        which = [0] * S
    else:
        pools = [gen.stream_pool(chunk_frames=chunk, sample_rate=r, pcm16=e == "pcm16") for r, e in FORMATS]
        which = [k % len(FORMATS) for k in range(S)]
    parts, first = [[] for _ in range(S)], [None] * S
    ticks, tick_start, handles = [], {}, {}
    pending = list(range(S))
    h = L.lib()
    torch.cuda.synchronize()
    n0, nbytes, t = h.fs2_kernel_launch_count(), 0, 0
    while pending or any(len(p) for p in pools):
        torch.cuda.synchronize()
        t0 = tick_start[t] = time.perf_counter()
        for k in [k for k in pending if arrive[k] <= t]:
            handles[(which[k], pools[which[k]].add(mels[k], sample_rate=fmt[k][0], encoding=fmt[k][1]))] = k
            pending.remove(k)
        produced = [(handles[(i, hd)], y) for i, p in enumerate(pools) for hd, _, y in p.step()]
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if produced:
            ticks.append((t1 - t0) * 1e3)
        for k, y in produced:
            if first[k] is None:
                first[k] = (t1 - tick_start[arrive[k]]) * 1e3
            parts[k].append(y)
            nbytes += y.numel() * y.element_size()
        t += 1
    launches = h.fs2_kernel_launch_count() - n0
    return ticks, first, [torch.cat(p, dim=2) for p in parts], launches, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--chunk", type=int, default=32)
    ap.add_argument("--gens", default="v1,v2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resample_mix_bench.py measures on a CUDA device; none is visible")
    print(json.dumps({"header": True, **gpu_info()}), flush=True)
    cfgs = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
    S, chunk = args.streams, args.chunk
    for g in args.gens.split(","):
        gen = generator(cfgs[g])
        _lens, arrive, mels = schedule(S, seed=100 + S)
        for arm in ARMS:                                   # warm-up: kernel setup, workspaces, tap uploads
            run(arm, gen, mels[:8], [0] * 8, chunk)
        res = {a: [] for a in ARMS}
        log, ref = [], None
        for r in range(args.rounds):
            for arm in ARMS:
                out = run(arm, gen, mels, arrive, chunk, log if arm == "mixed" and r == args.rounds - 1 else None)
                if ref is None:
                    ref = out[2]
                assert all(torch.equal(a, b) for a, b in zip(out[2], ref)), (g, arm)
                res[arm].append(out)
        torch.cuda.synchronize()
        conv = [(a.elapsed_time(b) * 1e3, n) for a, b, n in log]
        for arm in ARMS:
            ticks = [x for o in res[arm] for x in o[0]]
            first = [x for o in res[arm] for x in o[1]]
            n_ticks = statistics.median(len(o[0]) for o in res[arm])
            line = {"gen": g, "S": S, "chunk_frames": chunk, "arm": arm, "formats": [f"{r}/{e}" for r, e in FORMATS],
                    "tick_ms_median": round(statistics.median(ticks), 3), "tick_ms_p90": round(pct(ticks, 0.9), 3),
                    "first_chunk_ms_median": round(statistics.median(first), 3), "first_chunk_ms_p90": round(pct(first, 0.9), 3),
                    "launches_per_tick": round(statistics.median(o[3] for o in res[arm]) / n_ticks, 1),
                    "d2h_bytes_per_tick": round(statistics.median(o[4] for o in res[arm]) / n_ticks),
                    "bit_equal_across_arms": True}
            if arm == "mixed" and conv:
                us = statistics.median(c[0] for c in conv)
                byts = statistics.median(c[1] for c in conv)
                bound = byts / HBM_BYTES_PER_S * 1e6
                line.update({"conversion_call_us_median": round(us, 2), "conversion_bytes_median": round(byts),
                             "hbm_bound_us": round(bound, 3), "share_of_hbm_bound": round(bound / us, 4)})
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
