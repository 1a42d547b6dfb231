"""A/B of two builds of libfs2b200.so inside one process (box-to-box noise is 10-20 %): the in-tree library against a second build
passed on the command line (e.g. the previous commit built into scratch_ab/, which is not tracked).  Same inputs, same packed
weights; every comparison must match bit for bit.

  1. host logic (no GPU needed): fs2_{encode,decode,vocoder}_workspace_bytes for the LJSpeech and LibriTTS model shapes; for V1, V2
     and tests/test_stream_vocoder_cpu.py's other generator under each of its policies, the vocoder's launch plans
     (fs2_vocoder_window_plan, record for record; the plan of [0, T) is fs2_vocoder_forward's launches), its ResBlock runs and its
     offline and streams workspace sizes.  The new library stages the streams' origins and lengths into two [B] int32 tables of the
     streams workspace, and its window workspace equals its streams workspace.
  2. whole forwards: every output of FastSpeech2 and Generator (forward, stream, stream_pool) under several tensor-core / vocoder
     policies, the kernel launch count and the per-class launches of fs2_profile_begin / fs2_profile_end.  The new library's window
     call issues one staging launch (class 3) more than the old one's: stream() is expected to launch one more kernel per chunk.
  3. the tensor-core conv: ragged cases and every epilogue mode, then per-layer timing.

usage: python scripts/ab_lib.py [old.so]
"""
import ctypes as C, copy, os, sys, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from fastspeech2_b200 import _lib as L, configs, packing, synth
from fastspeech2_b200.spec import fastspeech2_spec


def bind(path):
    handle = C.CDLL(path)
    for name, (res, args) in L.EXPORTS.items():
        fn = getattr(handle, name, None)               # an older build may lack entry points this script does not call
        if fn is not None:
            fn.restype, fn.argtypes = res, args
    # the two builds may differ in ABI version; the structs this script passes must have the same layout in both
    for i, cls in ((0, L.Conv1dArgs), (9, L.AcousticModel), (10, L.EncodeArgs), (11, L.DecodeArgs), (12, L.VocoderModel), (13, L.VocoderArgs)):
        assert handle.fs2_struct_size(i) == C.sizeof(cls), (path, cls.__name__)
    return handle


old_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "scratch_ab", "libfs2b200_old.so")
libs = {"new": bind(L.LIB_PATH), "old": bind(old_path)}
SCRATCH = tempfile.mkdtemp()
DEFAULT_TC_MASK = L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8 | L.TC_ENCODER | L.TC_PREDICTORS

# ---------------------------------------------------------------------------------------------- 1. workspace sizes (host logic only)
def acoustic_shape(dataset, tc_mask, frame_level=False):
    pc, mc = configs.make_configs(dataset, SCRATCH)
    tr, vp = mc["transformer"], mc["variance_predictor"]
    m = L.AcousticModel(d_model=tr["encoder_hidden"], n_head=tr["encoder_head"], d_inner=tr["conv_filter_size"],
                        k1=tr["conv_kernel_size"][0], k2=tr["conv_kernel_size"][1], n_enc=tr["encoder_layer"], n_dec=tr["decoder_layer"],
                        n_mel=pc["preprocessing"]["mel"]["n_mel_channels"], vp_filter=vp["filter_size"], vp_kernel=vp["kernel_size"],
                        n_bins=mc["variance_embedding"]["n_bins"], tc_mask=tc_mask,
                        pitch_frame_level=int(frame_level), energy_frame_level=int(frame_level))
    post = [p for p in fastspeech2_spec(pc, mc) if p.key.startswith("postnet.convolutions.") and p.key.endswith(".0.conv.weight")]
    m.n_postnet = len(post)
    for i, p in enumerate(post):                       # Conv1d weight [cout][cin][k]
        m.post_cout[i], m.post_cin[i], m.post_k = p.shape
    return m


def vocoder_shape():
    h = configs.HIFIGAN_CONFIG
    m = L.VocoderModel(n_mel=h["num_mels"], c0=h["upsample_initial_channel"], n_stages=len(h["upsample_rates"]),
                       n_kernels=len(h["resblock_kernel_sizes"]), n_dil=len(h["resblock_dilation_sizes"][0]))
    for i, (u, k) in enumerate(zip(h["upsample_rates"], h["upsample_kernel_sizes"])):
        m.rates[i], m.up_k[i] = u, k
    for j, (k, dils) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
        m.rb_k[j] = k
        for d, dv in enumerate(dils):
            m.rb_dil[j][d] = dv
    return m


# (B, L) of BASELINE.json configs 0-4 and B = 1 / T = 7; decoder and vocoder T on both sides of 128 (fused attention from 128 on)
BATCHES, PHONEMES, FRAMES = (1, 16, 64), (7, 64, 128, 256), (7, 127, 128, 129, 1011, 1024, 2006)
n_ws = 0
for dataset in ("LJSpeech", "LibriTTS"):
    for tc_mask in (DEFAULT_TC_MASK, DEFAULT_TC_MASK & ~(L.TC_ENCODER | L.TC_PREDICTORS), 0):
        for frame_level in (False, True):
            m = acoustic_shape(dataset, tc_mask, frame_level)
            for B in BATCHES:
                for n in PHONEMES:
                    ws = {k: lib.fs2_encode_workspace_bytes(C.byref(m), B, n) for k, lib in libs.items()}
                    assert ws["new"] == ws["old"] > 0, ("encode", dataset, tc_mask, B, n, ws)
                for n in FRAMES:
                    ws = {k: lib.fs2_decode_workspace_bytes(C.byref(m), B, n) for k, lib in libs.items()}
                    assert ws["new"] == ws["old"] > 0, ("decode", dataset, tc_mask, B, n, ws)
                n_ws += len(PHONEMES) + len(FRAMES)
vm = vocoder_shape()
for B in BATCHES:
    for n in FRAMES:
        ws = {k: lib.fs2_vocoder_workspace_bytes(C.byref(vm), B, n) for k, lib in libs.items()}
        assert ws["new"] == ws["old"] > 0, ("vocoder", B, n, ws)
        n_ws += 1
print(f"workspace bytes: new == old for {n_ws} (model, B, L / T) queries", flush=True)

from tests.test_stream_vocoder_cpu import CONFIGS, POLICIES as PLAN_POLICIES, _model, _windows


def host(fn):
    """fn() through the package binding on each library."""
    got = {}
    for name, lib in libs.items():
        L._lib = lib
        got[name] = fn(lib)
    L._lib = None
    return got


n_plans = n_ws = 0
for cfg, shape in CONFIGS.items():
    for policy in PLAN_POLICIES:
        vm, _ = _model(shape, policy)
        for T in (1, 5, 40, 101, 1011):
            for f0, f1 in _windows(T) + [(0, T)]:
                if 0 <= f0 < T and f1 > f0:
                    got = host(lambda lib: [bytes(l) for l in L.vocoder_window_plan(vm, T, f0, f1)])
                    assert got["new"] == got["old"], ("window plan", cfg, policy, T, f0, f1)
                    n_plans += 1
        got = host(lambda lib: [[bytes(r) for r in L.vocoder_resblock_runs(vm, i)] for i in range(vm.n_stages)])
        assert got["new"] == got["old"], ("resblock runs", cfg, policy)
        for B in (1, 3, 16):
            for n in (1, 7, 64, 127, 1011):
                got = host(lambda lib: [f(C.byref(vm), B, n) for f in (lib.fs2_vocoder_workspace_bytes, lib.fs2_vocoder_streams_workspace_bytes,
                                                                      lib.fs2_vocoder_window_workspace_bytes)])
                tables = 2 * ((4 * B + 255) // 256 * 256)
                assert got["new"][:2] == [got["old"][0], got["old"][1] + tables] and min(got["new"]) > 0, ("vocoder workspaces", cfg, policy, B, n, got)
                assert got["new"][2] == got["new"][1], ("window workspace == streams workspace", cfg, policy, B, n, got)
                n_ws += 3
print(f"vocoder host logic: new == old for {n_plans} window plans and the ResBlock runs; {n_ws} workspace queries as expected", flush=True)
if not torch.cuda.is_available():
    print("no GPU: skipping the forward and conv sections")
    sys.exit(0)

# ---------------------------------------------------------------------------------------------- 2. whole forwards
from fastspeech2_b200.hifigan import AttrDict, Generator
from fastspeech2_b200.model import FastSpeech2

DEV = "cuda"


def same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    return a == b


def ab(label, fn, extra=0):
    """Run fn() once on each library (through the package binding) and assert identical outputs, and identical launches but for
    `extra` more class-3 launches in the new library."""
    got = {}
    for name in ("old", "new"):
        lib = libs[name]
        L._lib = lib
        fn()                                           # warm-up: workspaces, first-use setup
        torch.cuda.synchronize()
        ms, flops, launches = (C.c_double * L.PROF_CLASSES)(), (C.c_double * L.PROF_CLASSES)(), (C.c_int64 * L.PROF_CLASSES)()
        n0 = lib.fs2_kernel_launch_count()
        L.check(lib.fs2_profile_begin(), "fs2_profile_begin")
        out = fn()
        L.check(lib.fs2_profile_end(ms, flops, launches), "fs2_profile_end")
        n = lib.fs2_kernel_launch_count() - n0
        out = out if isinstance(out, tuple) else (out,)
        got[name] = (out, n, list(launches))
    (o_old, n_old, c_old), (o_new, n_new, c_new) = got["old"], got["new"]
    assert len(o_old) == len(o_new) and all(same(a, b) for a, b in zip(o_old, o_new)), f"{label}: outputs differ"
    assert n_old + extra == n_new, f"{label}: launch count {n_old} (old) vs {n_new} (new), expected {extra} more"
    assert [c + (extra if k == 3 else 0) for k, c in enumerate(c_old)] == c_new, f"{label}: per-class launches {c_old} (old) vs {c_new} (new)"
    print(f"{label:58s} identical, {n_new} launches, per class {c_new}", flush=True)


def fastspeech2(dataset, seed, frame_level=False):
    pc, mc = configs.make_configs(dataset, SCRATCH)
    if frame_level:
        pc = copy.deepcopy(pc)
        pc["preprocessing"]["pitch"]["feature"] = pc["preprocessing"]["energy"]["feature"] = "frame_level"
    m = FastSpeech2(pc, mc)
    m.load_state_dict(synth.fastspeech2_state_dict(pc, mc, seed=seed))
    return m.to(DEV).eval()


def on_dev(batch):
    spk, texts, lens, Lm = batch
    return spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm


lj = fastspeech2("LJSpeech", seed=0)
lj_batch = on_dev(synth.make_batch(16, 128, seed=0))
for label, mask in (("default tc_mask", DEFAULT_TC_MASK), ("TC_ENCODER | TC_PREDICTORS cleared", DEFAULT_TC_MASK & ~(L.TC_ENCODER | L.TC_PREDICTORS)),
                    ("tc_mask = 0", 0), ("F8 bits cleared", DEFAULT_TC_MASK & ~(L.TC_DECODER_F8 | L.TC_POSTNET_F8))):
    lj.tc_mask = mask
    lj.repack()
    ab(f"FastSpeech2 LJSpeech B16 x 128, {label}", lambda: lj(*lj_batch))
lj.tc_mask = DEFAULT_TC_MASK
lj.repack()
lj_out = lj(*lj_batch)

libri = fastspeech2("LibriTTS", seed=9)
libri_batch = on_dev(synth.make_batch(64, 256, seed=11, n_speakers=904, min_len=64))
ab("FastSpeech2 LibriTTS B64 ragged 64-256, multi-speaker", lambda: libri(*libri_batch))
del libri

frame = fastspeech2("LJSpeech", seed=15, frame_level=True)
frame_batch = on_dev(synth.make_batch(16, 128, seed=16, min_len=21))
ab("FastSpeech2 frame-level pitch / energy B16 x 128", lambda: frame(*frame_batch, p_control=1.1))
del frame

g = torch.Generator().manual_seed(5)
spk, texts, lens, Lm = synth.make_batch(4, 48, seed=6, min_len=15)
d_t = torch.randint(0, 3, (4, Lm), generator=g) * (torch.arange(Lm)[None, :] < lens[:, None])
mel_lens = d_t.sum(1)
T = int(mel_lens.max())
assert T < 128, T
p_t, e_t = torch.randn(4, Lm, generator=g), torch.randn(4, Lm, generator=g)
tf = tuple(t.to(DEV) for t in (spk, texts, lens)) + (Lm, None, mel_lens.to(DEV), T, p_t.to(DEV), e_t.to(DEV), d_t.to(DEV))
ab(f"FastSpeech2 teacher-forced B4, max_mel_len {T} < 128", lambda: lj(*tf))

POLICIES = {                                           # tests/test_gpu_ragged_vocoder.py
    "default": {},
    "fused_64ch_stage": {"fused_mask": 0b1100},
    "no_pairs": {"pair_mask": 0},
    "split3_everywhere": {"f8_mask": 0},
    "fp32_cuda_cores": {"use_tensor_cores": False},
}
mel_cl = lj_out[1].transpose(1, 2)                     # [B, 80, T] channels-last view of postnet_mel
mel_c = mel_cl.contiguous()                            # [B, 80, T] contiguous: the Generator transposes it first
ml = lj_out[9]


def generator(config, seed, **attrs):
    h = AttrDict(config)
    gen = Generator(h)
    gen.load_state_dict(synth.hifigan_state_dict(h, seed=seed))
    gen.eval()
    gen.remove_weight_norm()
    gen = gen.to(DEV)
    for k, v in attrs.items():
        setattr(gen, k, v)
    gen._invalidate()
    return gen


def pool_run(gen):
    """Three utterances through a stream pool of 32-frame chunks, the third admitted after the first step: each one's chunks, joined."""
    pool, chunks = gen.stream_pool(chunk_frames=32), {}
    mels = [mel_c[b, :, :int(ml[b])] for b in range(3)]
    pool.add(mels[0]), pool.add(mels[1])
    first = True
    while len(pool):
        for h, _, w in pool.step():
            chunks.setdefault(h, []).append(w)
        if first:
            pool.add(mels[2])
            first = False
    return tuple(torch.cat(chunks[h], -1) for h in sorted(chunks))


for policy, attrs in list(POLICIES.items()) + [("wide_pairs", {"wide_pairs": True})]:
    gen = generator(configs.HIFIGAN_CONFIG, 0, **attrs)
    for layout, mel in (("channels-last", mel_cl), ("contiguous", mel_c)):
        ab(f"Generator {policy}, {layout}, padded", lambda: gen(mel))
        ab(f"Generator {policy}, {layout}, ragged", lambda: gen(mel, mel_lens=ml))
    del gen
gen = generator(configs.HIFIGAN_V2_CONFIG, 1)
ab("Generator V2, padded", lambda: gen(mel_c))
ab("Generator V2, ragged", lambda: gen(mel_c, mel_lens=ml))
del gen
gen = generator(configs.HIFIGAN_CONFIG, 0)
ab("Generator stream(chunk_frames=64), ragged", lambda: torch.cat([w for _, w in gen.stream(mel_c, mel_lens=ml, chunk_frames=64)], -1),
   extra=-(-mel_c.shape[2] // 64))                    # the staging launch of every window
ab("Generator stream_pool(chunk_frames=32), 3 streams", lambda: pool_run(gen))
del gen
L._lib = None
print("whole forwards: new == old bit for bit, same launches", flush=True)

# ---------------------------------------------------------------------------------------------- 3. tensor-core conv
stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)


def run(lib, x, w, wtc, y, *, bias=None, k=1, dil=1, res=None, acc=False, lens=None, in_act=0, out_act=0, alpha=1.0):
    B, T, Cin = x.shape
    N = w.shape[2]
    a = L.Conv1dArgs(x=x.data_ptr(), x_batch_stride=x.stride(0), x_row_stride=x.stride(1), B=B, T=T, Cin=Cin, w=w.data_ptr(), bias=L.ptr(bias),
                     N=N, taps=k, dilation=dil, pad_left=(k - 1) * dil // 2, w_tc=wtc.data_ptr(), backend=L.CONV_TC, tc_variant=0,
                     in_act=in_act, in_slope=0.1, out_act=out_act, out_slope=0.1, res=L.ptr(res),
                     res_batch_stride=res.stride(0) if res is not None else 0, res_row_stride=res.stride(1) if res is not None else 0,
                     alpha=alpha, accumulate=int(acc), row_lens=L.ptr(lens), y=y.data_ptr(), y_batch_stride=y.stride(0), y_row_stride=y.stride(1))
    rc = lib.fs2_conv1d(C.byref(a), stream)
    assert rc == 0, rc


g = torch.Generator().manual_seed(0)
# correctness first: ragged / partial tiles / every epilogue mode, new == old bit for bit
for (B, T, Cin, N, k, dil, res, acc, in_act, out_act) in ((3, 300, 64, 96, 3, 1, True, True, 3, 0), (2, 1000, 256, 256, 5, 1, True, False, 0, 2), (5, 77, 32, 32, 7, 3, False, False, 3, 3),
                                                           (2, 515, 128, 64, 11, 5, False, True, 3, 1), (1, 129, 80, 512, 5, 1, True, True, 0, 0), (2, 700, 256, 80, 1, 1, False, False, 0, 0),
                                                           (4, 2051, 32, 32, 3, 1, True, False, 3, 0), (2, 4100, 64, 64, 7, 1, True, True, 3, 0)):
    x = (torch.randn(B, T, Cin, generator=g) * 3).cuda(); r = torch.randn(B, T, N, generator=g).cuda() if res else None
    lens = torch.randint(1, T + 1, (B,), generator=g).int().cuda()
    w = torch.randn(k, Cin, N, generator=g) * (k * Cin) ** -0.5
    b = torch.randn(N, generator=g).cuda()
    wtc = packing.pack_conv_tc(w).cuda(); w = w.cuda()
    outs = {}
    for name, lib in libs.items():
        y = torch.full((B, T, N), 0.25, device="cuda")
        run(lib, x, w, wtc, y, bias=b, k=k, dil=dil, res=r, acc=acc, lens=lens, in_act=in_act, out_act=out_act, alpha=0.5)
        torch.cuda.synchronize()
        outs[name] = y
    assert torch.equal(outs["new"], outs["old"]), (B, T, Cin, N, k, (outs["new"] - outs["old"]).abs().max().item())
print("conv: new == old bit for bit on ragged cases", flush=True)

CASES = (("s0 C256 k3", 256, 256, 3, 1, 8192, False, False), ("s0 C256 k7 res", 256, 256, 7, 1, 8192, True, False), ("s0 C256 k11", 256, 256, 11, 5, 8192, False, False),
         ("s1 C128 k3", 128, 128, 3, 1, 65536, False, False), ("s1 C128 k3 res", 128, 128, 3, 1, 65536, True, False), ("s1 C128 k7", 128, 128, 7, 3, 65536, False, False),
         ("s1 C128 k11 res+acc", 128, 128, 11, 1, 65536, True, True), ("s2 C64 k3", 64, 64, 3, 1, 131072, False, False), ("s2 C64 k7 res", 64, 64, 7, 1, 131072, True, False),
         ("s2 C64 k11 res+acc", 64, 64, 11, 1, 131072, True, True), ("s3 C32 k3", 32, 32, 3, 1, 262144, False, False), ("s3 C32 k7 res", 32, 32, 7, 1, 262144, True, False),
         ("s3 C32 k11 res+acc", 32, 32, 11, 1, 262144, True, True), ("ups1 C256->512 k2", 256, 512, 2, 1, 8192, False, False), ("ups3 C64->32 k2", 64, 32, 2, 1, 131072, False, False),
         ("dec ffn1 k9", 256, 1024, 9, 1, 1024, False, False), ("dec ffn2 k1 res", 1024, 256, 1, 1, 1024, True, False), ("dec qkv", 256, 768, 1, 1, 1024, False, False),
         ("postnet k5", 512, 512, 5, 1, 1024, False, False))
tot = {"new": 0.0, "old": 0.0}
for name, Cin, N, k, dil, T, res, acc in CASES:
    x = torch.randn(16, T, Cin, generator=g).cuda(); r = torch.randn(16, T, N, generator=g).cuda() if res else None
    w = torch.randn(k, Cin, N, generator=g) * (k * Cin) ** -0.5
    wtc = packing.pack_conv_tc(w).cuda(); w = w.cuda()
    y = torch.zeros(16, T, N, device="cuda")
    best = {"new": 1e9, "old": 1e9}
    for rep in range(3):
        for which in ("old", "new"):
            lib = libs[which]
            run(lib, x, w, wtc, y, k=k, dil=dil, res=r, acc=acc, in_act=3); torch.cuda.synchronize()
            for _ in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); run(lib, x, w, wtc, y, k=k, dil=dil, res=r, acc=acc, in_act=3); e1.record(); torch.cuda.synchronize()
                best[which] = min(best[which], e0.elapsed_time(e1) * 1e3)
    for kx in tot: tot[kx] += best[kx]
    print(f"{name:22s} old {best['old']:7.1f} us | new {best['new']:7.1f} us | {100 * (best['new'] / best['old'] - 1):+6.1f} %", flush=True)
print(f"sum: old {tot['old']:.0f} us, new {tot['new']:.0f} us, {100 * (tot['new'] / tot['old'] - 1):+.1f} %")
