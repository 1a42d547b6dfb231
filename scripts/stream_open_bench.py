"""Open streams of the vocoder pool (StreamPool.open / feed / close): mel that arrives in pieces, against streams added whole.

  (a) pool: S streams (S = 16 and 64) of LJSpeech-like lengths (1012 +- 150 mel frames, seeded) arriving over the first 8 ticks, V1
      and V2, 32-frame chunks.  Two arms, alternating:
        open: each stream opened on arrival and fed 8 frames per tick (a view of its mel, no copy), closed after its last block;
        add:  each stream added whole on arrival (Generator.stream_pool as before).
      tick_ms median / p90: host clock around one tick that produced audio, ending in a device synchronise (the open arm's streams
      join every fourth tick or so: 8 frames arrive per tick, a chunk takes 32).  launches_per_tick: fs2_kernel_launch_count over those
      ticks.  first_chunk_ms median / p90: from the start of a stream's arrival tick to the end of the tick that produced its first
      chunk (the open arm waits for the chunk's cone: 32 + 14 frames, 6 ticks of feeding).  Every stream's waveform is checked bit for
      bit across the arms.
  (b) long form: a paragraph of 10 synthetic sentences (synth.make_batch, 40-120 phonemes, seeded), FastSpeech2 (LJSpeech config,
      ragged) then V1 or V2 through one open stream of 32-frame chunks.  Two arms, alternating:
        batch:    one FastSpeech2 call on the 10 sentences, then each sentence's postnet_mel[b, :n].T fed in order;
        sentence: one FastSpeech2 call per sentence, its mel fed as it returns, the pool stepped until nothing more is ready.
      first_audio_ms: host clock from the start to the end of the step that produced the first chunk; total_ms: to the last chunk.
      The open stream is checked bit for bit against the vocoder's forward on the joined mel; whether the arms' waveforms are equal
      (ragged FastSpeech2 synthesises each sentence of a batch as alone) is reported.
      seam_max_abs: max |difference| between the open stream and the 10 sentences added as separate streams and joined, within the
      vocoder's receptive field (reach frames) of each sentence boundary; away_max_abs: the same elsewhere (0: the seam is all there is).

Prints a header line with the GPU name, power limit and max SM clock, then one JSON line per (part, generator, S / arm).

usage: python scripts/stream_open_bench.py [--rounds 3] [--streams 16,64] [--gens v1,v2] [--parts a,b]
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from fastspeech2_b200 import _lib as L, configs, synth  # noqa: E402
from fastspeech2_b200.hifigan.models import mel_reach  # noqa: E402
from fastspeech2_b200.model import FastSpeech2  # noqa: E402
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from stream_pool_bench import pct, schedule  # noqa: E402
from stream_vocoder_bench import generator, gpu_info  # noqa: E402

CHUNK, BLOCK = 32, 8


def run_pool(arm, gen, mels, arrive):
    """(ms of each tick that produced audio, per-stream first-chunk ms, per-stream waveform, launches over those ticks)."""
    S = len(mels)
    pool = gen.stream_pool(chunk_frames=CHUNK)
    parts, first, tick_start, ticks = [[] for _ in range(S)], [None] * S, {}, []
    handles, fed, pending = {}, {}, list(range(S))
    h = L.lib()
    launches, t = 0, 0
    while pending or len(pool):
        torch.cuda.synchronize()
        n0, t0 = h.fs2_kernel_launch_count(), time.perf_counter()
        tick_start[t] = t0
        for k in [k for k in pending if arrive[k] <= t]:
            pending.remove(k)
            if arm == "add":
                handles[pool.add(mels[k])] = k
            else:
                hd = pool.open()
                handles[hd], fed[k] = k, (hd, 0)
        for k, (hd, a) in list(fed.items()):
            n = mels[k].shape[1]
            pool.feed(hd, mels[k][:, a:a + BLOCK])
            fed[k] = (hd, a + BLOCK)
            if a + BLOCK >= n:
                pool.close(hd)
                del fed[k]
        produced = [(handles[hd], w) for hd, _, w in pool.step()]
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        if produced:
            ticks.append((t1 - t0) * 1e3)
            launches += h.fs2_kernel_launch_count() - n0
        for k, w in produced:
            if first[k] is None:
                first[k] = (t1 - tick_start[arrive[k]]) * 1e3
            parts[k].append(w)
        t += 1
    return ticks, first, [torch.cat(p, dim=2) for p in parts], launches


def part_a(g, gen, streams, rounds):
    for S in streams:
        lens, arrive, mels = schedule(S, seed=100 + S)
        run_pool("open", gen, mels[:2], [0, 0])                  # warm-up: kernel setup, workspaces, pinned blocks
        res = {"open": [], "add": []}
        ref = None
        for _ in range(rounds):
            for arm in ("open", "add"):
                ticks, first, wavs, launches = run_pool(arm, gen, mels, arrive)
                ref = ref or wavs
                assert all(torch.equal(a, b) for a, b in zip(wavs, ref)), (g, S, arm)
                res[arm].append((ticks, first, launches))
        for arm, rs in res.items():
            ticks = [x for r in rs for x in r[0]]
            first = [x for r in rs for x in r[1]]
            print(json.dumps({
                "part": "a", "gen": g, "S": S, "chunk_frames": CHUNK, "block_frames": BLOCK, "arm": arm,
                "tick_ms_median": round(statistics.median(ticks), 3), "tick_ms_p90": round(pct(ticks, 0.9), 3),
                "audio_ticks": round(statistics.median(len(r[0]) for r in rs)),
                "launches_per_tick": round(sum(r[2] for r in rs) / len(ticks), 1),
                "first_chunk_ms_median": round(statistics.median(first), 3), "first_chunk_ms_p90": round(pct(first, 0.9), 3),
                "bit_equal_across_arms": True}), flush=True)


def acoustic():
    pc, mc = configs.make_configs("LJSpeech", tempfile.mkdtemp())
    model = FastSpeech2(pc, mc)
    model.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=0))
    return model.to("cuda").eval()


def run_long(arm, model, gen, batch):
    """(first-audio ms, total ms, waveform [1, 1, N], per-sentence frames)."""
    spk, texts, lens, Lmax = (x.to("cuda") if torch.is_tensor(x) else x for x in batch)
    lens_h = batch[2].tolist()
    pool = gen.stream_pool(chunk_frames=CHUNK)
    parts, first = [], None
    torch.cuda.synchronize()
    t0 = time.perf_counter()

    def drain():
        nonlocal first
        while True:
            out = pool.step()
            if not out:
                return
            parts.append(out[0][2])
            if first is None:
                torch.cuda.synchronize()
                first = (time.perf_counter() - t0) * 1e3
    hd = pool.open()
    frames = []
    if arm == "batch":
        out = model(spk, texts, lens, Lmax, ragged=True)
        ns = out[9].tolist()
        for b, n in enumerate(ns):
            pool.feed(hd, out[1][b, :n].T)
        frames = ns
        pool.close(hd)
        drain()
    else:
        for b, n_b in enumerate(lens_h):
            out = model(spk[b:b + 1], texts[b:b + 1, :n_b], lens[b:b + 1], n_b, ragged=True)
            n = int(out[9][0])
            pool.feed(hd, out[1][0, :n].T)
            frames.append(n)
            if b == len(lens_h) - 1:
                pool.close(hd)
            drain()
    torch.cuda.synchronize()
    return first, (time.perf_counter() - t0) * 1e3, torch.cat(parts, dim=2), frames, out


def part_b(g, gen, model, rounds):
    batch = synth.make_batch(10, 120, seed=7, min_len=40)
    up = gen._pack()[3]
    run_long("batch", model, gen, batch)
    run_long("sentence", model, gen, batch)
    res = {"batch": [], "sentence": []}
    ref, equal = None, True
    for _ in range(rounds):
        for arm in res:
            first, total, wav, frames, _ = run_long(arm, model, gen, batch)
            ref = ref if ref is not None else (wav, frames)
            equal = equal and frames == ref[1] and torch.equal(wav, ref[0])
            res[arm].append((first, total))
    # the seam: the sentences' mels (from the one-call arm) as separate add()ed streams, joined, against the open stream
    spk, texts, lens, Lmax = batch
    out = model(spk.cuda(), texts.cuda(), lens.cuda(), Lmax, ragged=True)
    frames = ref[1]
    mels = [out[1][b, :n].T for b, n in enumerate(frames)]
    joined = torch.cat(mels, dim=1)
    assert torch.equal(ref[0], gen(joined[None])), "open stream against forward on the joined mel"
    pool = gen.stream_pool(chunk_frames=CHUNK)
    hs = [pool.add(m) for m in mels]
    sep = {h: [] for h in hs}
    while len(pool):
        for h, _, w in pool.step():
            sep[h].append(w)
    separate = torch.cat([torch.cat(sep[h], dim=2) for h in hs], dim=2)
    diff = (separate - ref[0]).abs()[0, 0]
    reach = max(mel_reach(gen._pack()[0], CHUNK)) * up
    near = torch.zeros_like(diff, dtype=torch.bool)
    edge = 0
    for n in frames[:-1]:
        edge += n * up
        near[max(edge - reach, 0):edge + reach] = True
    for arm, rs in res.items():
        print(json.dumps({
            "part": "b", "gen": g, "arm": arm, "sentences": len(frames), "frames": sum(frames), "chunk_frames": CHUNK,
            "first_audio_ms_median": round(statistics.median(r[0] for r in rs), 3),
            "total_ms_median": round(statistics.median(r[1] for r in rs), 3),
            "first_audio_ms_rounds": [round(r[0], 3) for r in rs], "total_ms_rounds": [round(r[1], 3) for r in rs],
            "seam_max_abs": float(diff[near].max()), "away_max_abs": float(diff[~near].max()), "seam_window_samples": reach,
            "bit_equal_across_arms": equal, "bit_equal_to_forward": True}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--streams", default="16,64")
    ap.add_argument("--gens", default="v1,v2")
    ap.add_argument("--parts", default="a,b")
    args = ap.parse_args()
    print(json.dumps({"header": True, **gpu_info()}), flush=True)
    cfgs = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}
    parts = args.parts.split(",")
    model = acoustic() if "b" in parts else None
    for g in args.gens.split(","):
        gen = generator(cfgs[g])
        if "a" in parts:
            part_a(g, gen, [int(s) for s in args.streams.split(",")], args.rounds)
        if "b" in parts:
            part_b(g, gen, model, args.rounds)


if __name__ == "__main__":
    main()
