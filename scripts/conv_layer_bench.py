"""Warm timings of single fs2_conv1d layers on the tensor-core kernel, grouped by epilogue: plain (LeakyReLU out), residual, and
residual + accumulate into y (the last conv of every ResBlock after the first), at the shapes the vocoder runs through per-layer
launches (stages 0 and 1 of HiFi-GAN V1: B = 16 x 1 017 mel frames, every kernel size and dilation, and the two stages'
ConvTranspose phase groups), plus the K-segmented convs of an encoder FFT block.  The same layer with and without the residual / accumulate input shows what reading those costs.

usage: python scripts/conv_layer_bench.py [--quick] [other.so ...]
  other.so: further builds of libfs2b200.so (same ABI) timed on the same inputs, alternating with the in-tree library
  --quick:  dilation 1 only"""
import ctypes as C, os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from fastspeech2_b200 import _lib as L, ops, packing

DEV = "cuda"
g = torch.Generator().manual_seed(0)
B, T0 = 16, 1017
quick = "--quick" in sys.argv


def bind(path):
    handle = C.CDLL(path)
    for name, (res, args) in L.EXPORTS.items():
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = res, args
    assert handle.fs2_abi_version() == L.ABI_VERSION, path
    return handle


libs = {"tree": L.lib()}
libs.update({os.path.basename(p): bind(p) for p in sys.argv[1:] if not p.startswith("--")})


def timed(fn, n):
    best = {}
    for _ in range(3):                                  # alternate the builds, keep each one's best mean over n launches
        for name, lib in libs.items():
            L._lib = lib
            fn(); torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n): fn()
            e1.record(); torch.cuda.synchronize()
            best[name] = min(best.get(name, 1e30), e0.elapsed_time(e1) * 1e3 / n)
    L._lib = libs["tree"]
    return best


def report(label, us, flops):
    cols = " | ".join(f"{name} {t:8.1f} us {flops / t / 1e6:6.1f} TFLOP/s" for name, t in us.items())
    print(f"{label:44s} {cols}", flush=True)


def vocoder_layer(stage, C, up, k, dil, f8, mode, n=10):
    """mode: 'plain' (LeakyReLU out, no residual), 'res' (+ residual), 'res+acc' (+ residual, alpha 1/3, added into y)"""
    N = T0 * up
    x = torch.randn(B, N, C, generator=g).to(DEV)
    w = torch.randn(k, C, C, generator=g) * (C * k) ** -0.5
    b = torch.randn(C, generator=g).to(DEV) * 0.05
    wt = packing.pack_conv_tc(w, f8=f8).to(DEV)
    wd = w.to(DEV)
    r = torch.randn(B, N, C, generator=g).to(DEV) if mode != "plain" else None
    acc = mode == "res+acc"
    y = torch.randn(B, N, C, generator=g).to(DEV) * 0.1
    fn = lambda: ops.conv1d(x, wd, b, dilation=dil, pad_left=(k - 1) * dil // 2, in_act=3, in_slope=0.1, out_act=0 if r is not None else 3,
                            out_slope=0.1, res=r, alpha=1 / 3 if acc else 1.0, accumulate=acc, out=y, w_tc=wt, backend=2,
                            tc_variant=1 if f8 else 0)
    report(f"s{stage} C={C:3d} k={k:2d} dil={dil} {'f16+f8' if f8 else 'split3':6s} {mode:7s}", timed(fn, n), 2.0 * B * N * C * C * k)


def upsample_group(stage, Cin, rows, rate, n=10):
    """one ConvTranspose1d phase group as the vocoder runs it: LeakyReLU in, 2 taps, Cin -> (rate / 2) * Cin / 2 channels at the stage's
    input rows (T0 * rows), f16 + f8"""
    T, N = T0 * rows, (rate // 2) * (Cin // 2)
    x = torch.randn(B, T, Cin, generator=g).to(DEV)
    w = torch.randn(2, Cin, N, generator=g) * (Cin * 2) ** -0.5
    b = torch.randn(N, generator=g).to(DEV) * 0.05
    wt = packing.pack_conv_tc(w, f8=True).to(DEV)
    wd = w.to(DEV)
    y = torch.empty(B, T, N, device=DEV)
    fn = lambda: ops.conv1d(x, wd, b, pad_left=1, in_act=3, in_slope=0.1, out=y, w_tc=wt, backend=2, tc_variant=1)
    report(f"s{stage} upsample group Cin={Cin} N={N} k=2 f16+f8", timed(fn, n), 2.0 * B * T * Cin * N * 2)


def segmented_layer(label, T, Cin, N, k, res, n=20):
    """K-segmented encoder conv (FS2_TC_VARIANT_NB64 | SEGMENTED): every (tap, 256-channel) slice is one work unit summed in fp32"""
    x = torch.randn(B, T, Cin, generator=g).to(DEV)
    w = torch.randn(k, Cin, N, generator=g) * (Cin * k) ** -0.5
    b = torch.randn(N, generator=g).to(DEV) * 0.05
    wt = packing.pack_conv_tc_segments(w).to(DEV)
    wd = w.to(DEV)
    r = torch.randn(B, T, N, generator=g).to(DEV) if res else None
    y = torch.empty(B, T, N, device=DEV)
    fn = lambda: ops.conv1d(x, wd, b, pad_left=(k - 1) // 2, in_act=3 if res else 0, in_slope=0.0, res=r, out=y, w_tc=wt, backend=2,
                            tc_variant=L.TC_VARIANT_NB64 | L.TC_VARIANT_SEGMENTED)
    report(f"{label:44s}"[:44], timed(fn, n), 2.0 * B * T * Cin * N * k)


print(f"device: {torch.cuda.get_device_name()}, builds: {', '.join(libs)}", flush=True)
for stage, C, up in ((0, 256, 8), (1, 128, 64)):
    for k in (3, 7, 11):
        for dil in ((1,) if quick else (1, 3, 5)):
            for mode in ("plain", "res", "res+acc"):
                vocoder_layer(stage, C, up, k, dil, True, mode)
for stage, Cin, rows in ((0, 512, 1), (1, 256, 8)):      # the ConvTranspose phase groups of stages 0 and 1 (rate 8 each)
    upsample_group(stage, Cin, rows, 8)
for mode in ("plain", "res", "res+acc"):                 # split-fp16 at 128 output channels per work item
    vocoder_layer(1, 128, 64, 11, 1, False, mode)
segmented_layer("enc ffn1 256->1024 k=9 segmented", 128, 256, 1024, 9, False)
segmented_layer("enc ffn2 1024->256 k=1 segmented res", 128, 1024, 256, 1, True)
segmented_layer("frame ffn2 1024->256 k=1 segmented res", 1024, 1024, 256, 1, True)
