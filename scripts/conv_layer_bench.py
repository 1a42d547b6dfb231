"""Warm timings of single HiFi-GAN-shaped fs2_conv1d layers on the tensor-core kernel (B = 16 x 1017 frames), both operand splits.
Usage: python scripts/conv_layer_bench.py [one]   (one = a single (C=128, k=3, f8) layer in a loop, for ncu)"""
import sys, os, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from fastspeech2_b200 import ops, packing
DEV = "cuda"
g = torch.Generator().manual_seed(0)
B, T0 = 16, 1017
one = len(sys.argv) > 1

def run(C, up, k, dil, f8, res, n=10):
    N = T0 * up
    x = torch.randn(B, N, C, generator=g).to(DEV)
    w = torch.randn(k, C, C, generator=g) * (C * k) ** -0.5
    b = torch.randn(C, generator=g).to(DEV) * 0.05
    wt = packing.pack_conv_tc(w, f8=f8).to(DEV)
    wd = w.to(DEV)
    r = torch.randn(B, N, C, generator=g).to(DEV) if res else None
    y = torch.empty_like(x)
    fn = lambda: ops.conv1d(x, wd, b, dilation=dil, pad_left=(k - 1) * dil // 2, in_act=3, in_slope=0.1, out_act=0 if res else 3, out_slope=0.1,
                            res=r, out=y, w_tc=wt, backend=2, tc_variant=1 if f8 else 0)
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    fl = 2.0 * B * N * C * C * k
    gb = (2 + (1 if res else 0)) * B * N * C * 4 / 1e9
    print(f"C={C:3d} rows={B*N:8d} k={k:2d} dil={dil} {'f16+f8' if f8 else 'split3':6s} res={int(res)}: {ms*1e3:7.1f} us  {fl/ms/1e9:6.1f} TFLOP/s  {gb/ms*1e3:5.0f} GB/s algorithmic", flush=True)

if one:
    run(128, 64, 3, 1, True, False, n=3)
    run(128, 64, 7, 1, True, False, n=3)
else:
    for C, up in ((256, 8), (128, 64), (64, 128)):
        for k in (3, 7, 11):
            for f8 in (True, False):
                run(C, up, k, 1, f8, False)
            run(C, up, k, 1, True, True)
