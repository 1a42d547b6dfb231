"""HiFi-GAN V2 against V1 at bench.py's configs[2] shape (B = 16 x 1012 mel frames), CUDA-event timed with a warm-up, modes alternating.

  vocoder:   V1 and V2 (default policies), padded and ragged (lengths spread over [T/2, T]); V2 with every ResBlock conv on per-layer
             launches (fused_mask = pair_mask = 0) and with use_tensor_cores = False.  Before timing, the three V2 policies must agree
             within the 1e-4 waveform bar.
  resstack:  each narrow V2 stage's ResBlock group (16 channels at 128 rows per frame, 8 channels at 256) as one fs2_resstack launch
             against its 18 per-layer fs2_conv1d launches (f16 + f8 tensor-core tiles at 16 channels, the exact kernel at 8).
  e2e:       FastSpeech2 (LJSpeech config, 16 x 128 phonemes as bench.py) followed by V2 through the public modules.

Prints one JSON line with ms per call (median over rounds) and the GPU name and power limit queried in the same run.

usage: python scripts/hifigan_v2_bench.py [--rounds 5] [--calls 5] [--warmup-s 1.0]
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
import torch  # noqa: E402

from fastspeech2_b200 import _lib as L, configs, ops, packing, synth  # noqa: E402
from fastspeech2_b200.hifigan import AttrDict, Generator  # noqa: E402
from fastspeech2_b200.model import FastSpeech2  # noqa: E402
from scripts.ragged_vocoder_bench import gpu_info, time_calls  # noqa: E402

DEV = "cuda"
B, T = 16, 1012
SHIPPED = ((3, 7, 11), ((1, 3, 5),) * 3)


def vocoder(cfg, seed, **policy):
    h = AttrDict(cfg)
    gen = Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=seed))
    gen.eval()
    with contextlib.redirect_stdout(io.StringIO()):
        gen.remove_weight_norm()
    for k, v in policy.items():
        setattr(gen, k, v)
    return gen.to(DEV)


def timed(modes, rounds, calls, warmup_s):
    """{name: median ms per call} of zero-argument callables, alternating in every round."""
    t_end = time.perf_counter() + warmup_s
    while time.perf_counter() < t_end:
        for fn in modes.values():
            fn()
    torch.cuda.synchronize()
    ms = {k: [] for k in modes}
    for _ in range(rounds):
        for k, fn in modes.items():
            ms[k].append(time_calls(fn, calls))
    return {k: round(statistics.median(v), 3) for k, v in ms.items()}


def resstack_group(C, rows_per_frame, seed):
    """(fused, per_layer) callables for one ResBlock group at C channels over B x T mel frames."""
    N = T * rows_per_frame
    g = lambda s: torch.Generator().manual_seed(s)
    x = (torch.randn(B, N, C, generator=g(seed))).to(DEV)
    w = lambda s, k: packing.conv_w(torch.randn(C, C, k, generator=g(s)) * 0.6 * (C * k) ** -0.5)
    ks, dils = SHIPPED
    w1 = [[w(seed + 10 * j + d, k) for d in range(3)] for j, k in enumerate(ks)]
    w2 = [[w(seed + 500 + 10 * j + d, k) for d in range(3)] for j, k in enumerate(ks)]
    b = [[(0.05 * torch.randn(C, generator=g(seed + 900 + 3 * j + d))).to(DEV) for d in range(3)] for j in range(3)]
    tiles = lambda v: (packing.pack_conv_tc_pad16(v) if C == 8 else packing.pack_conv_tc(v, f8=True)).to(DEV)
    t1, t2 = [[tiles(v) for v in r] for r in w1], [[tiles(v) for v in r] for r in w2]
    w1d, w2d = [[v.to(DEV) for v in r] for r in w1], [[v.to(DEV) for v in r] for r in w2]
    y, r1, r2, tmp = (torch.empty_like(x) for _ in range(4))
    per_layer_tc = C % 16 == 0

    def conv(src, j, d, second, dst, res=None, alpha=1.0, acc=False):
        k, dil = ks[j], 1 if second else dils[j][d]
        wd, wt = (w2d, t2) if second else (w1d, t1)
        ops.conv1d(src, wd[j][d], b[j][d], dilation=dil, pad_left=(k - 1) * dil // 2, in_act=L.ACT_LRELU, in_slope=0.1,
                   out_act=L.ACT_NONE if second else L.ACT_LRELU, out_slope=0.1, res=res, alpha=alpha, out=dst, accumulate=acc,
                   w_tc=wt[j][d] if per_layer_tc else None, backend=L.CONV_TC if per_layer_tc else L.CONV_SIMT,
                   tc_variant=1 if per_layer_tc else 0)

    def per_layer():                 # model.cu's unfused vocoder path
        for j in range(3):
            r = x
            for d in range(3):
                last = d == 2
                dst = y if last else (r2 if r is r1 else r1)
                conv(r, j, d, False, tmp)
                conv(tmp, j, d, True, dst, res=r, alpha=1.0 / 3 if last else 1.0, acc=last and j > 0)
                r = dst
        return y

    fused = lambda: ops.resstack(x, ks, dils, t1, b, t2, b, out=y)
    return fused, per_layer


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--warmup-s", type=float, default=1.0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hifigan_v2_bench.py measures on the GPU; no CUDA device is visible")
    out = {"shape": f"B={B} x T={T} mel frames", **gpu_info()}
    mel = synth.make_mel(B, T, seed=3).to(DEV)
    lens = torch.linspace(T // 2, T, B).round().long().to(DEV)
    v1 = vocoder(configs.HIFIGAN_CONFIG, 1)
    v2 = {"default": vocoder(configs.HIFIGAN_V2_CONFIG, 1),
          "per_layer": vocoder(configs.HIFIGAN_V2_CONFIG, 1, fused_mask=0, pair_mask=0),
          "fp32": vocoder(configs.HIFIGAN_V2_CONFIG, 1, use_tensor_cores=False)}
    with torch.no_grad():
        ref = v2["fp32"](mel)
        out["v2_policy_max_abs_diff"] = {k: (g(mel) - ref).abs().max().item() for k, g in v2.items() if k != "fp32"}
    assert all(v < 1e-4 for v in out["v2_policy_max_abs_diff"].values()), out["v2_policy_max_abs_diff"]

    modes = {"v1_padded": lambda: v1(mel), "v1_ragged": lambda: v1(mel, mel_lens=lens),
             "v2_padded": lambda: v2["default"](mel), "v2_ragged": lambda: v2["default"](mel, mel_lens=lens),
             "v2_per_layer": lambda: v2["per_layer"](mel), "v2_fp32": lambda: v2["fp32"](mel)}
    out["vocoder_ms"] = timed(modes, args.rounds, args.calls, args.warmup_s)
    del v1, v2
    torch.cuda.empty_cache()

    groups = {}
    for C, rpf in ((16, 128), (8, 256)):
        fused, per_layer = resstack_group(C, rpf, seed=40 + C)
        groups[f"C{C}_fused_1_launch"], groups[f"C{C}_per_layer_18_launches"] = fused, per_layer
    out["resblock_group_ms"] = timed(groups, args.rounds, args.calls, args.warmup_s)
    del groups
    torch.cuda.empty_cache()

    pc, mc = configs.make_configs("LJSpeech", tempfile.mkdtemp())
    model = FastSpeech2(pc, mc)
    model.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=0))
    model = model.to(DEV).eval()
    voc = vocoder(configs.HIFIGAN_V2_CONFIG, 1)
    spk, texts, slens, Lmax = (t.to(DEV) if torch.is_tensor(t) else t for t in synth.make_batch(B, 128, seed=0))

    def e2e():
        with torch.no_grad():
            o = model(spk, texts, slens, Lmax)
            return voc(o[1].transpose(1, 2), mel_lens=o[9])
    out["fs2_v2_e2e_ms"] = timed({"fs2+v2": e2e}, args.rounds, args.calls, args.warmup_s)["fs2+v2"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
