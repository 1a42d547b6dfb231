"""Time each fused HiFi-GAN ResBlock stage under the whole-group launch and under the run planner's launches
(fs2_vocoder_resblock_runs), and the whole Generator.forward, for V1 and V2 at bench.py's configs[2] shape (B = 16 x 1012 mel frames),
padded and ragged (lengths spread over [T/2, T]).  CUDA-event timed after a warm-up, modes alternating in every round.

  stages:      per fused stage, the group launch and the planned runs on the Generator's packed weights; both must agree bit for bit
               (on the rows below each utterance's length when ragged) before they are timed.
  candidates:  (--candidates) every cut of each ResBlock's dilations into consecutive runs, timed alone (padded): the data the
               planner's cost model is fitted to.
  forward:     Generator.forward with this library, and with --old-lib PATH also with a second build of libfs2b200.so (e.g. the
               parent commit's), alternating in the same process; the two waveforms must be equal bit for bit.

Prints readable lines and one JSON line with ms per call (median over rounds) and the GPU name and power limit queried in the same run.

usage: python scripts/resblock_runs_bench.py [--candidates] [--old-lib PATH] [--rounds 5] [--calls 5] [--warmup-s 1.0]
"""
import argparse
import ctypes as C
import itertools
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from fastspeech2_b200 import _lib as L, configs, synth  # noqa: E402
from scripts.hifigan_v2_bench import timed, vocoder  # noqa: E402
from scripts.ragged_vocoder_bench import gpu_info  # noqa: E402
from tests.test_gpu_resblock_runs import run_stage  # noqa: E402

DEV = "cuda"
B, T = 16, 1012
CONFIGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG}


class Stage:
    """Stage i's ResBlock group of a packed Generator on a random [B][T * rows per frame][C] input."""

    def __init__(self, gen, i, seed):
        m, pk, _, _ = gen._packed or gen._pack()
        self.m, self.pk, self.i = m, pk, i
        self.nk, self.nd = m.n_kernels, m.n_dil
        self.C = m.c0 >> (i + 1)
        self.scale = 1
        for u in range(i + 1):
            self.scale *= m.rates[u]
        N = T * self.scale
        self.ks = [m.rb_k[j] for j in range(self.nk)]
        self.dils = [[m.rb_dil[j][d] for d in range(self.nd)] for j in range(self.nk)]
        g = torch.Generator().manual_seed(seed)
        self.x = (0.5 * torch.randn(B, N, self.C, generator=g)).to(DEV)
        self.y, self.r1, self.r2 = (torch.empty_like(self.x) for _ in range(3))
        self.runs = [(r.j, r.d0, r.d1) for r in L.vocoder_resblock_runs(m, i)]

    def launch(self, runs, lens=None):
        """The launches of `runs` [(j, d0, d1)] (j = -1: the whole group), as fs2_vocoder_forward issues them; returns y."""
        return run_stage(self.m, self.pk, self.i, self.x, lens, runs, (self.y, self.r1, self.r2))

    def cuts(self, j):
        """Every cut of ResBlock j's dilations into consecutive runs: {label: [(j, d0, d1), ...]}"""
        out = {}
        for ends in itertools.product((False, True), repeat=self.nd - 1):
            bounds = [0] + [d + 1 for d, e in enumerate(ends) if e] + [self.nd]
            runs = [(j, a, b) for a, b in zip(bounds, bounds[1:])]
            out["|".join(",".join(str(self.dils[j][d]) for d in range(a, b)) for _, a, b in runs)] = runs
        return out


def fused_stages(gen):
    _, fused, _, _ = gen.effective_masks()
    return [i for i in range(gen.num_upsamples) if (fused >> i) & 1]


def bind(path):
    """A second build of the library, bound like scripts/ab_lib.py does (that script runs on import): the structs passed to it must
    have this binding's layout."""
    handle = C.CDLL(path)
    for name, (res, args) in L.EXPORTS.items():
        fn = getattr(handle, name, None)
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    for i, cls in ((12, L.VocoderModel), (13, L.VocoderArgs)):
        assert handle.fs2_struct_size(i) == C.sizeof(cls), (path, cls.__name__)
    return handle


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--candidates", action="store_true")
    ap.add_argument("--old-lib", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup-s", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resblock_runs_bench.py measures on the GPU; no CUDA device is visible")
    out = {"shape": f"B={B} x T={T} mel frames", **gpu_info()}
    print(out, flush=True)
    mel = synth.make_mel(B, T, seed=3).to(DEV)
    lens = torch.linspace(T // 2, T, B).round().int().to(DEV)
    out["stages"], out["candidates"], out["forward_ms"] = {}, {}, {}
    for name, cfg in CONFIGS.items():
        gen = vocoder(cfg, 1)
        for i in fused_stages(gen):
            st = Stage(gen, i, seed=10 + i)
            tag = f"{name}_stage{i}_C{st.C}"
            group = [(-1, 0, st.nd)]
            for lab, ln in (("padded", None), ("ragged", lens)):
                a = st.launch(group, ln).clone()
                b = st.launch(st.runs, ln).clone()
                if ln is None:
                    assert torch.equal(a, b), tag
                else:
                    n = (lens.long() * st.scale).tolist()
                    assert all(torch.equal(a[u, :n[u]], b[u, :n[u]]) for u in range(B)), tag
            ms = timed({"group_padded": lambda: st.launch(group), "runs_padded": lambda: st.launch(st.runs),
                        "group_ragged": lambda: st.launch(group, lens), "runs_ragged": lambda: st.launch(st.runs, lens)},
                       args.rounds, args.calls, args.warmup_s)
            out["stages"][tag] = {"runs": st.runs, **ms}
            print(f"{tag}: runs {st.runs}\n    {ms}", flush=True)
            if args.candidates:
                modes = {f"j{j}_k{st.ks[j]}[{lab}]": (lambda r=r: st.launch(r)) for j in range(st.nk) for lab, r in st.cuts(j).items()}
                modes["group"] = lambda: st.launch(group)
                cms = timed(modes, args.rounds, args.calls, args.warmup_s)
                out["candidates"][tag] = cms
                print(f"    candidates {cms}", flush=True)
            del st
            torch.cuda.empty_cache()
        libs = {"new": L.lib()}
        if args.old_lib:
            libs["old"] = bind(args.old_lib)

        wide = vocoder(cfg, 1, wide_pairs=True) if gen._stages_of_width(128) else None

        def fwd(which, ln):
            L._lib = libs["new" if which == "wide_pairs" else which]
            return (wide if which == "wide_pairs" else gen)(mel, mel_lens=ln)
        for lab, ln in (("padded", None), ("ragged", lens)):
            if "old" in libs:
                assert torch.equal(fwd("old", ln), fwd("new", ln)), (name, lab)
            modes = list(libs) + (["wide_pairs"] if wide is not None else [])
            if wide is not None:
                out.setdefault("wide_pairs_max_abs_diff", {})[f"{name}_{lab}"] = (fwd("wide_pairs", ln) - fwd("new", ln)).abs().max().item()
            ms = timed({f"{w}": (lambda w=w, ln=ln: fwd(w, ln)) for w in modes}, args.rounds, args.calls, args.warmup_s)
            out["forward_ms"][f"{name}_{lab}"] = ms
            print(f"{name} forward {lab}: {ms}", flush=True)
        L._lib = libs["new"]
        del gen, wide
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
