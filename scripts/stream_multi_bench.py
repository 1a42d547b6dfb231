"""Streams of several HiFi-GAN generators: one multi-generator pool (Generator.stream_pool(generators=...)) against one pool per
generator, and a one-generator pool on fs2_vocoder_forward_streams against the same streams through fs2_vocoder_forward_streams_multi
with n_models = 1 (what the per-item weight-pointer and header loads cost).

Workload: 64 streams of ~1012 mel frames (980..1043) arrive over 8 ticks (8 per tick), chunk_frames = 32, stream k on generator
k % G, G = 2 and 4 synthetic generators of V1 and of V2.  Arms alternate, three rounds; per arm: tick median and p90 (host clock
around each tick, which ends in a device synchronise), launches per tick (fs2_kernel_launch_count), first-chunk latency after
arrival (from the tick's start at which a stream is added to the end of the tick that returns its first chunk), median and p90, and
whether every stream is bit-identical across arms.  Prints one JSON line per (config, G) with the card and its power limit.

    python scripts/stream_multi_bench.py [--rounds 3] [--configs v1,v2] [--gens 2,4]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastspeech2_b200 import _lib as L, configs, synth  # noqa: E402
from fastspeech2_b200.hifigan import AttrDict, Generator  # noqa: E402

DEV = "cuda"
N_STREAMS, ARRIVAL_TICKS, CHUNK = 64, 8, 32
CFGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}


def _generator(cfg, seed):
    h = AttrDict(cfg)
    g = Generator(h)
    g.load_state_dict(synth.hifigan_state_dict(h, seed=seed))
    g.eval()
    g.remove_weight_norm()
    return g.to(DEV)


def _run(pools, mels, which):
    """Drives `pools` (stream k goes to pools[pool_of[k]] with generator index gen_of[k]) over the arrival schedule.  Returns tick
    times (s), launches per tick, first-chunk latencies (s) and each stream's concatenated output."""
    lib = L.lib()
    arrive = [k // (N_STREAMS // ARRIVAL_TICKS) for k in range(N_STREAMS)]
    handles, parts, added_at, first = {}, {}, {}, {}
    ticks, launches = [], []
    tick = 0
    while tick < ARRIVAL_TICKS or any(len(p) for p in pools):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n0 = lib.fs2_kernel_launch_count()
        for k in range(N_STREAMS):
            if arrive[k] == tick:
                p, g = which(k)
                handles[(p, pools[p].add(mels[k], generator=g))] = k
                added_at[k] = t0
        done = []
        for p, pool in enumerate(pools):
            for h, _, chunk in pool.step():
                done.append((handles[(p, h)], chunk))
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        ticks.append(t1 - t0)
        launches.append(lib.fs2_kernel_launch_count() - n0)
        for k, chunk in done:
            parts.setdefault(k, []).append(chunk)
            first.setdefault(k, t1 - added_at[k])
        tick += 1
    return ticks, launches, [first[k] for k in range(N_STREAMS)], {k: torch.cat(v, dim=-1) for k, v in parts.items()}


def _stats(ticks, launches, first):
    ms = lambda v, q: round(float(np.percentile(np.asarray(v) * 1e3, q)), 3)
    return {"tick_ms_median": ms(ticks, 50), "tick_ms_p90": ms(ticks, 90), "launches_per_tick": round(float(np.mean(launches)), 1),
            "first_chunk_ms_median": ms(first, 50), "first_chunk_ms_p90": ms(first, 90)}


def _one_model_multi(pool):
    """The pool's own launch call, but through fs2_vocoder_forward_streams_multi with n_models = 1."""
    launch = pool._launch
    pool._launch = lambda ptrs, f0s, ns, caps=None: launch(ptrs, f0s, ns, caps, gens=[0] * len(ptrs))
    return pool


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default="v1,v2")
    ap.add_argument("--gens", default="2,4")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("stream_multi_bench.py needs a CUDA device")
    card = torch.cuda.get_device_name()
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                               timeout=30).stdout.strip().splitlines()[0]
    except Exception:                                   # noqa: BLE001 -- the card is still named
        power = "unknown"
    rng = np.random.default_rng(0)
    for cfg in args.configs.split(","):
        for G in (int(g) for g in args.gens.split(",")):
            gens = [_generator(CFGS[cfg], seed=100 + i) for i in range(G)]
            mels = [synth.make_mel(1, int(rng.integers(980, 1044)), seed=k)[0].to(DEV) for k in range(N_STREAMS)]
            arms = {
                "multi_pool": lambda: ([gens[0].stream_pool(CHUNK, generators=gens[1:])], lambda k: (0, k % G)),
                "pool_per_generator": lambda: ([g.stream_pool(CHUNK) for g in gens], lambda k: (k % G, 0)),
                "one_generator_streams": lambda: ([gens[0].stream_pool(CHUNK)], lambda k: (0, 0)),
                "one_generator_multi_n1": lambda: ([_one_model_multi(gens[0].stream_pool(CHUNK))], lambda k: (0, 0)),
            }
            for make in arms.values():                  # warm-up: module loads, workspaces, every shape of the timed runs
                pools, which = make()
                _run(pools, mels, which)
            res = {a: {"ticks": [], "launches": [], "first": []} for a in arms}
            outs = {}
            for _ in range(args.rounds):
                for a, make in arms.items():            # alternating arms, round by round
                    pools, which = make()
                    t, n, f, out = _run(pools, mels, which)
                    res[a]["ticks"] += t
                    res[a]["launches"] += n
                    res[a]["first"] += f
                    prev = outs.setdefault(a, out)
                    assert all(torch.equal(prev[k], out[k]) for k in range(N_STREAMS))
            same_multi = all(torch.equal(outs["multi_pool"][k], outs["pool_per_generator"][k]) for k in range(N_STREAMS))
            same_n1 = all(torch.equal(outs["one_generator_streams"][k], outs["one_generator_multi_n1"][k]) for k in range(N_STREAMS))
            line = {"config": cfg, "generators": G, "streams": N_STREAMS, "chunk_frames": CHUNK, "rounds": args.rounds, "card": card,
                    "power_limit": power, "bit_identical_multi_vs_per_generator": same_multi,
                    "bit_identical_streams_vs_multi_n1": same_n1}
            for a in arms:
                line[a] = _stats(res[a]["ticks"], res[a]["launches"], res[a]["first"])
            print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
