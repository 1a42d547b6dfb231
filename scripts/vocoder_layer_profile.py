"""Per-launch breakdown of one HiFi-GAN V1 forward at the bench step's shape (configs[2]: B = 16 x 1 012 mel frames, padded), grouped
by stage and layer kind.  Kernel times come from torch.profiler (CUDA activity) over several forwards, matched record for record to
fs2_vocoder_window_plan(m, T, 0, T), which lists forward's launches in order.  Per group: median time per forward, share of the
forward, algorithmic TFLOP/s and the least HBM traffic (every input row read once, every output row written once, the residual and
the accumulated y read once) over time.

usage: python scripts/vocoder_layer_profile.py [--lib other.so] [--reps N]
  --lib: time another build of libfs2b200.so (same ABI) instead of the in-tree one"""
import argparse, collections, contextlib, ctypes as C, io, os, statistics, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.hifigan import AttrDict, Generator

ap = argparse.ArgumentParser()
ap.add_argument("--lib", default=None)
ap.add_argument("--reps", type=int, default=5)
args = ap.parse_args()
if args.lib:
    handle = C.CDLL(args.lib)
    for name, (res, argtypes) in L.EXPORTS.items():
        fn = getattr(handle, name)
        fn.restype, fn.argtypes = res, argtypes
    assert handle.fs2_abi_version() == L.ABI_VERSION, args.lib
    L._lib = handle

B, T = 16, 1012
dev = torch.device("cuda:0")
h = AttrDict(configs.HIFIGAN_CONFIG)
voc = Generator(h)
voc.load_state_dict(synth.hifigan_state_dict(h, seed=0))
voc.eval()
with contextlib.redirect_stdout(io.StringIO()):
    voc.remove_weight_norm()
voc.to(dev)
mel = synth.make_mel(B, T, seed=0).to(dev)
for _ in range(3):
    voc(mel)
torch.cuda.synchronize()
plan = L.vocoder_window_plan(voc._packed[0], T, 0, T)

with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(args.reps):
        voc(mel)
    torch.cuda.synchronize()
# the plan's launches (conv and ResBlock kernels), not the transpose of the [B, 80, T] mel or torch's own kernels
kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and ("conv" in e.name or "resstack" in e.name)]
kernels.sort(key=lambda e: e.time_range.start)
assert len(kernels) == args.reps * len(plan), (len(kernels), len(plan))

KIND = {L.VW_CONV_PRE: "conv_pre", L.VW_UP_A: "upsample", L.VW_UP_B: "upsample", L.VW_RB_CONV1: "resblock conv1",
        L.VW_RB_CONV2: "resblock conv2", L.VW_RB_PAIR: "resblock pair", L.VW_RB_GROUP: "resblock fused run", L.VW_CONV_POST: "conv_post"}
c0, rates = h.upsample_initial_channel, h.upsample_rates


def traffic(r):
    """least HBM bytes of launch r: input rows x input channels, output rows x output channels, + residual and accumulated y"""
    s = r.stage
    if r.layer == L.VW_CONV_PRE:
        cin, cout = 80, c0
    elif r.layer in (L.VW_UP_A, L.VW_UP_B):
        cin, cout = c0 >> s, rates[s] // 2 * (c0 >> (s + 1))
    elif r.layer == L.VW_CONV_POST:
        cin, cout = c0 >> len(rates), 1
    else:
        cin = cout = c0 >> (s + 1)
    extra = 0
    if r.layer == L.VW_RB_CONV2:
        extra = (2 if r.j > 0 and r.d == len(h.resblock_dilation_sizes[r.j]) - 1 else 1) * cout
    return 4.0 * B * ((r.x1 - r.x0) * cin + (r.y1 - r.y0) * (cout + extra))


per = [statistics.median(kernels[k * len(plan) + i].time_range.elapsed_us() for k in range(args.reps)) for i in range(len(plan))]
groups = collections.OrderedDict()
for r, us in zip(plan, per):
    key = ("-" if r.stage < 0 else str(r.stage), KIND[r.layer])
    g = groups.setdefault(key, [0, 0.0, 0.0, 0.0])
    g[0] += 1; g[1] += us; g[2] += B * r.flops; g[3] += traffic(r)          # the plan's FLOPs are per utterance
total = sum(per)
print(f"device: {torch.cuda.get_device_name()}, build: {L.lib().fs2_build_info().decode()}, {args.reps} forwards, B = {B} x {T} frames")
print(f"forward (sum of kernel times): {total / 1e3:.2f} ms over {len(plan)} launches")
print(f"{'stage':5s} {'layer':20s} {'launches':>8s} {'ms':>8s} {'share':>6s} {'TFLOP/s':>8s} {'TB/s':>6s}")
for (stage, kind), (n, us, fl, by) in groups.items():
    print(f"{stage:5s} {kind:20s} {n:8d} {us / 1e3:8.3f} {100 * us / total:5.1f}% {fl / us / 1e6:8.1f} {by / us / 1e6:6.2f}")
