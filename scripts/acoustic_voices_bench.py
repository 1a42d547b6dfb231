"""Several FastSpeech2 voices in one acoustic call: one VoiceBank call against one FastSpeech2.forward call per voice on the same
utterances, padded and ragged.  The one-voice rows measure what the voices mode's per-item weight-pointer loads cost against forward.

Workload: LJSpeech config, G = 1, 2, 4, 8 voices from synthetic seeds (voice 2's pitch / energy bins scaled, as another stats.json
gives), U = 1 and 4 utterances per voice of 128 phonemes (about 1 000 frames each), voice of utterance k = k % G.  Both arms compute
every utterance's mel; the per-voice arm's calls each end in forward's host synchronise for the output length, as a server's would.
Arms alternate within each of --rounds rounds of --iters calls; per arm: the median of the call times (CUDA events around the host
calls, which end in a device synchronise), and the launches per call (fs2_kernel_launch_count).  Prints one JSON line per (G, U,
mode) with the card and its power limit.

    python scripts/acoustic_voices_bench.py [--rounds 5] [--iters 5] [--voices 1,2,4,8] [--per-voice 1,4]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastspeech2_b200 import _lib as L, configs, synth  # noqa: E402
from fastspeech2_b200.model import FastSpeech2, VoiceBank  # noqa: E402

DEV = "cuda"
PHONEMES = 128


def _voice(cfgs, seed, bins):
    pc, mc = cfgs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=seed)
    for k in ("variance_adaptor.pitch_bins", "variance_adaptor.energy_bins"):
        sd[k] = sd[k] * bins
    m = FastSpeech2(pc, mc)
    m.load_state_dict(sd)
    return m.to(DEV).eval()


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def _timed(fn, iters):
    """Median ms of `iters` calls of fn (CUDA events around each), and the launches of one call"""
    lib = L.lib()
    times = []
    for _ in range(iters):
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n0 = lib.fs2_kernel_launch_count()
        a.record()
        fn()
        b.record()
        b.synchronize()
        n = lib.fs2_kernel_launch_count() - n0
        times.append(a.elapsed_time(b))
    return times, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--voices", default="1,2,4,8")
    ap.add_argument("--per-voice", default="1,4")
    args = ap.parse_args()
    cfgs = configs.make_configs("LJSpeech", tempfile.mkdtemp(prefix="fs2cfg"))
    gs = [int(g) for g in args.voices.split(",")]
    models = [_voice(cfgs, 70 + k, 1.07 if k == 2 else 1.0) for k in range(max(gs))]
    card = _card()
    for G in gs:
        for U in (int(u) for u in args.per_voice.split(",")):
            B = G * U
            spk, texts, lens, Lm = synth.make_batch(B, PHONEMES, seed=80 + B, min_len=PHONEMES)
            spk, texts, lens = spk.to(DEV), texts.to(DEV), lens.to(DEV)
            voice = torch.tensor([k % G for k in range(B)])
            rows = [torch.tensor([b for b in range(B) if b % G == k], device=DEV) for k in range(G)]
            bank = VoiceBank(models[:G])
            for ragged in (False, True):
                arms = {
                    "bank": lambda: bank(voice, spk, texts, lens, Lm, ragged=ragged),
                    "per_voice": lambda: [models[k](spk[r], texts[r], lens[r], Lm, ragged=ragged) for k, r in enumerate(rows)],
                }
                for fn in arms.values():                 # warm: packing, workspaces, position tables, module loads
                    fn()
                times = {k: [] for k in arms}
                launches = {}
                for _ in range(args.rounds):
                    for name, fn in arms.items():
                        t, launches[name] = _timed(fn, args.iters)
                        times[name] += t
                frames = int(bank(voice, spk, texts, lens, Lm, ragged=ragged)[9].sum())
                print(json.dumps({"voices": G, "per_voice": U, "B": B, "phonemes": PHONEMES, "frames": frames,
                                  "mode": "ragged" if ragged else "padded",
                                  "bank_ms": round(float(np.median(times["bank"])), 3),
                                  "per_voice_ms": round(float(np.median(times["per_voice"])), 3),
                                  "bank_launches": launches["bank"], "per_voice_launches": launches["per_voice"],
                                  "card": card}), flush=True)


if __name__ == "__main__":
    main()
