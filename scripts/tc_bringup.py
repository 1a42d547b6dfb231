"""GPU bring-up of the tensor-core conv kernel: every case runs in its own subprocess (a wedged kernel cannot take the
rest down) for each descriptor variant; prints max-abs error against an fp64 CPU evaluation of the fs2_conv1d contract."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {
    # name: (B, T, Cin, N, taps, dil, pad, in_act, out_act, res, alpha, acc, lens)
    "k1_c16_n128_t128": (1, 128, 16, 128, 1, 1, 0, 0, 0, 0, 1.0, 0, 0),
    "k1_c64_n128_t128": (1, 128, 64, 128, 1, 1, 0, 0, 0, 0, 1.0, 0, 0),
    "k3_c64_n128_t128": (1, 128, 64, 128, 3, 1, 1, 0, 0, 0, 1.0, 0, 0),
    "k3_c64_n128_t300_b2": (2, 300, 64, 128, 3, 1, 1, 0, 0, 0, 1.0, 0, 0),
    "k11d5_c128_n128_t700": (2, 700, 128, 128, 11, 5, 25, 3, 3, 1, 1.0, 0, 0),
    "k7_c256_n256_t520_acc": (2, 520, 256, 256, 7, 1, 3, 0, 0, 1, 1.0 / 3, 1, 0),
    "k5_c512_n80_res": (2, 333, 512, 80, 5, 1, 2, 0, 0, 1, 1.0, 0, 0),
    "k9_c256_n1024_relu": (2, 260, 256, 1024, 9, 1, 4, 0, 1, 0, 1.0, 0, 0),
    "k1_c1024_n256_res_mask": (3, 200, 1024, 256, 1, 1, 0, 0, 0, 1, 1.0, 0, 1),
    "k3d3_c32_n32": (2, 1500, 32, 32, 3, 3, 3, 3, 3, 0, 1.0, 0, 0),
    "k7_c80_n512": (2, 150, 80, 512, 7, 1, 3, 0, 0, 0, 1.0, 0, 0),
    "k2_c64_n64_up": (2, 257, 64, 64, 2, 1, 1, 3, 0, 0, 1.0, 0, 0),
}


def run_case(name, variant):
    import torch
    from fastspeech2_b200 import ops, packing
    from tests import emul_cabi as E
    B, T, Cin, N, taps, dil, pad, in_act, out_act, use_res, alpha, acc, use_lens = CASES[name]
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, Cin, generator=g)
    w = torch.randn(taps, Cin, N, generator=g) * (taps * Cin) ** -0.5
    bias = torch.randn(N, generator=g) * 0.1
    res = torch.randn(B, T, N, generator=g) if use_res else None
    y0 = torch.randn(B, T, N, generator=g) if acc else None
    lens = torch.tensor([max(1, T - 7 * (i + 1)) for i in range(B)], dtype=torch.int32) if use_lens else None
    d = lambda t: None if t is None else t.double()
    want = E.conv1d(x.double(), w.double(), bias.double(), dil, pad, in_act, 0.1, out_act, 0.1, d(res), alpha, d(y0), lens)
    dev = "cuda"
    c = lambda t: None if t is None else t.to(dev)
    wtc = packing.pack_conv_tc(w)
    out = {}
    for label, kw in (("simt", dict(backend=1)), ("tc", dict(backend=2, w_tc=c(wtc), tc_variant=variant))):
        y = c(y0).clone() if acc else None
        got = ops.conv1d(c(x), c(w), c(bias), dilation=dil, pad_left=pad, in_act=in_act, in_slope=0.1, out_act=out_act, out_slope=0.1,
                         res=c(res), alpha=alpha, out=y, accumulate=bool(acc), row_lens=c(lens), **kw)
        torch.cuda.synchronize()
        err = (got.cpu().double() - want).abs()
        out[label] = dict(max=float(err.max()), mean=float(err.mean()), nan=bool(torch.isnan(got).any()))
    out["scale"] = float(want.abs().max())
    print("RESULT " + json.dumps(out))


if __name__ == "__main__":
    if len(sys.argv) >= 3:
        run_case(sys.argv[1], int(sys.argv[2]))
        sys.exit(0)
    for variant in (0,):
        bad = 0
        for name in CASES:
            try:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), name, str(variant)], capture_output=True, text=True,
                                   timeout=120)
                line = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
                if line:
                    res = json.loads(line[0][7:])
                    ok = res["tc"]["max"] < 2e-5 * max(1.0, res["scale"]) and not res["tc"]["nan"]
                    bad += 0 if ok else 1
                    print(f"variant {variant} {name:28s} tc max {res['tc']['max']:.3e} mean {res['tc']['mean']:.3e} | simt max "
                          f"{res['simt']['max']:.3e} | scale {res['scale']:.2f} {'OK' if ok else 'BAD'}", flush=True)
                else:
                    bad += 1
                    print(f"variant {variant} {name:28s} FAILED rc={r.returncode}: {(r.stderr or r.stdout)[-400:]}", flush=True)
            except subprocess.TimeoutExpired:
                bad += 1
                print(f"variant {variant} {name:28s} TIMEOUT (kernel wedged)", flush=True)
                if name == "k1_c16_n128_t128":
                    break
        print(f"variant {variant}: {bad} bad", flush=True)
        if bad == 0:
            break
