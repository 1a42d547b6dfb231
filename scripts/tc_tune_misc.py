"""Tune the tensor-core conv kernel inside ONE process: taps per weight stage (TPS) and weight ring depth per HiFi-GAN layer shape.
Debug hook fs2_debug_set_tc_tuning(sa, sb, tps, grid) (library built with FS2_DEBUG_KNOBS=1; 0 = the heuristic's choice)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fastspeech2_b200 import _lib, ops, packing
lib = _lib.lib()
lib.fs2_debug_set_tc_tuning.argtypes = [ctypes.c_int] * 4
g = torch.Generator().manual_seed(0)
shapes = [("s3 C32 k3", 32, 32, 3, 1, 262144, False), ("s3 C32 k7 res", 32, 32, 7, 1, 262144, True), ("s2 C64 k3", 64, 64, 3, 1, 131072, False),
          ("s2 C64 k7 res", 64, 64, 7, 1, 131072, True), ("s2 C64 k11", 64, 64, 11, 1, 131072, False), ("ups3 C64->32 k2", 64, 32, 2, 1, 131072, False),
          ("ups2 C128->64 k2", 128, 64, 2, 1, 65536, False), ("s1 C128 k3", 128, 128, 3, 1, 65536, False), ("s1 C128 k7", 128, 128, 7, 1, 65536, False),
          ("s1 C128 k11", 128, 128, 11, 1, 65536, False), ("s0 C256 k3", 256, 256, 3, 1, 8192, False), ("s0 C256 k7", 256, 256, 7, 1, 8192, False)]
settings = [("default", (0, 0, 0, 0)), ("tps1", (0, 0, 1, 0)), ("tps2", (0, 0, 2, 0)), ("tps3", (0, 0, 3, 0)), ("tps4", (0, 0, 4, 0)), ("tps6", (0, 0, 6, 0)),
            ("sb2", (0, 2, 0, 0)), ("sb3", (0, 3, 0, 0)), ("sb6", (0, 6, 0, 0)), ("default", (0, 0, 0, 0))]
for name, Cin, N, k, dil, T, res in shapes:
    B = 16
    x = torch.randn(B, T, Cin, generator=g).cuda()
    w = torch.randn(k, Cin, N, generator=g) * (k * Cin) ** -0.5
    wtc = packing.pack_conv_tc(w).cuda(); w = w.cuda()
    r = torch.randn(B, T, N, generator=g).cuda() if res else None
    kw = dict(dilation=dil, pad_left=(k * dil - dil) // 2, w_tc=wtc, backend=2, res=r, in_act=3, in_slope=0.1)
    line = f"{name:18s}"
    for label, st in settings:
        lib.fs2_debug_set_tc_tuning(*st)
        try:
            ops.conv1d(x, w, None, **kw); torch.cuda.synchronize()
            ts = []
            for _ in range(4):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); ops.conv1d(x, w, None, **kw); e1.record(); torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
            line += f" | {label}: {min(ts):4.0f}"
        except Exception as ex:
            line += f" | {label}:  n/a"
    lib.fs2_debug_set_tc_tuning(0, 0, 0, 0)
    print(line, flush=True)
