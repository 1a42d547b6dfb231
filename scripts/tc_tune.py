"""A/B the tensor-core conv kernel's ring depths / taps-per-stage inside ONE process (box-to-box noise is ~10-20 %)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from fastspeech2_b200 import _lib, ops, packing
lib = _lib.lib()
lib.fs2_debug_set_tc_tuning.argtypes = [ctypes.c_int] * 4
g = torch.Generator().manual_seed(0)
shapes = [("s1 C128 k3", 128, 128, 3, 1, 65536, False), ("s1 C128 k3 res", 128, 128, 3, 1, 65536, True), ("s1 C128 k11", 128, 128, 11, 1, 65536, False),
          ("s3 C32 k3", 32, 32, 3, 1, 262144, False), ("s3 C32 k11 res", 32, 32, 11, 1, 262144, True), ("s2 C64 k7", 64, 64, 7, 1, 131072, False),
          ("s0 C256 k7", 256, 256, 7, 1, 8192, False), ("s2 C64 k11 res", 64, 64, 11, 1, 131072, True), ("dec ffn1 256->1024 k9", 256, 1024, 9, 1, 1012, False), ("postnet 512->512 k5", 512, 512, 5, 1, 1012, False)]
settings = [(0, 0, 1), (0, 0, 3), (0, 0, 4), (0, 4, 4), (0, 3, 6), (0, 2, 6), (0, 2, 8), (0, 2, 11), (0, 3, 11), (3, 2, 11)]
for name, Cin, N, k, dil, T, res in shapes:
    B = 16
    x = torch.randn(B, T, Cin, generator=g).cuda()
    w = torch.randn(k, Cin, N, generator=g) * (k * Cin) ** -0.5
    wtc = packing.pack_conv_tc(w).cuda(); w = w.cuda()
    r = torch.randn(B, T, N, generator=g).cuda() if res else None
    kw = dict(dilation=dil, pad_left=(k * dil - dil) // 2, w_tc=wtc, backend=2, res=r)
    line = f"{name:24s}"
    for (sa, sb, tps) in settings:
        lib.fs2_debug_set_tc_tuning(sa, sb, tps, 0)
        try:
            ops.conv1d(x, w, None, **kw); torch.cuda.synchronize()
            ts = []
            for _ in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); ops.conv1d(x, w, None, **kw); e1.record(); torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1) * 1e3)
            line += f" | sa{sa} sb{sb} tps{tps}: {min(ts):6.0f}"
        except Exception as ex:
            line += f" | sa{sa} sb{sb} tps{tps}:   n/a"
    lib.fs2_debug_set_tc_tuning(0, 0, 0, 0)
    print(line, flush=True)
