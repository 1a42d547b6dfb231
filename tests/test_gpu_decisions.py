"""GPU: the kernels that make FastSpeech2's discrete decisions, and the vocoder's conv_post, against fp64 and the reference's semantics.

  - fs2_variance_head: the prediction per element against fp64 within its rounding depth; the bucket exactly torch.bucketize of the
    kernel's own fp32 key (edges, their fp32 neighbours, +-0, subnormals, +-inf, NaN), on the prediction path under scalar controls and
    on the target path; the embedding add bit for bit;
  - fs2_durations: d_rounded against fp64 round(exp(s) - 1) * c, and cum / mel_lens / len_stats exactly from the kernel's own d;
  - fs2_length_regulate: exactly a gather, T below, at and above the total;
  - the per-element control instantiations through FastSpeech2.forward (fs2_acoustic_encode_ctl), padded and ragged: NaN and inf
    controls reach the buckets and the durations as in the reference;
  - fs2_conv_post, both kernels, against fp64 within each kernel's summation depth."""
import math

import pytest
import torch

from fastspeech2_b200 import _lib as L, ops, synth
from fastspeech2_b200.model import FastSpeech2
from oracle import fs2_oracle as O
from tests.test_decisions_cpu import BINS, bucket_keys, same

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                    # fp32 unit roundoff
FLT_MAX = 3.4028234663852886e38
MEL_TOL = 1e-3                    # tests/test_gpu_model.py's mel bar


def gamma(n):
    return n * U / (1 - n * U)


def ulp32(v):
    """Spacing of fp32 at |v| (v: float64 tensor of finite values)."""
    a = v.abs().float()
    return (torch.nextafter(a, torch.tensor(math.inf)) - a).double()


def rnd(*shape, seed, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def _index_emb(n_edges, D=4):
    return torch.arange(n_edges + 1, dtype=torch.float32)[:, None].repeat(1, D)


# ------------------------------------------------------------------------------------------------------------ variance head: prediction
def head_depth(C):
    """Rounding depth n of variance_head_kernel's prediction: a product h*w is rounded once (1), added to its float4 pair partner (1),
    the two pairs are added (1), the float4 sum joins the lane's accumulator once per lane iteration, ceil(C / 128) of them, then the
    5-level warp_sum (5), the bias add (1) and the control multiply (1).  So every product passes through at most n = 10 + ceil(C / 128)
    roundings, the bias through at most 7, and |pred - pred64| <= gamma_n * (sum |h*w| + |b|) * |c| (Higham, Accuracy and Stability,
    eq. 3.5, applied to a summation tree of that depth; FMA contraction only removes roundings)."""
    return 10 + (C // 4 + 31) // 32


def _cancelling(h, w, rows):
    """Rows whose products cancel pairwise up to fp32 rounding: h[j] * w[j] = -h[j + C/2] * w[j + C/2]."""
    C = w.numel()
    p = h[rows, :C // 2] * w[:C // 2]
    h[rows, :C // 2] = p / w[:C // 2]
    h[rows, C // 2:] = -p / w[C // 2:]


@pytest.mark.parametrize("scale", [2.0 ** -12, 1.0, 2.0 ** 8])
@pytest.mark.parametrize("C,Lm", [(4, 13), (128, 29), (256, 45), (1024, 19)])
def test_variance_head_prediction_against_fp64(C, Lm, scale, parity_log):
    """pred = (h . w + b) * c per element within gamma_n (sum |h*w| + |b|) |c|, n = head_depth(C); rows past lens[b] are 0 * c exactly.
    B * L is not a multiple of the kernel's 8 rows per block; rows 3 and 4 of every utterance cancel."""
    B = 3
    h = rnd(B, Lm, C, seed=C, scale=scale)
    w = rnd(C, seed=C + 1, scale=0.1)
    w[w.abs() < 1e-3] = 1e-3
    b = torch.tensor([0.3 * scale])
    for bb in range(B):
        _cancelling(h[bb], w, [3, 4])
    lens = torch.tensor([Lm, Lm // 2, 1], dtype=torch.int32)
    pad = torch.arange(Lm)[None, :] >= lens[:, None].long()
    worst = 0.0
    for c in (1.0, 1.3, -1.0):
        bins = torch.linspace(-1.0, 1.0, 7).to(DEV)
        got = ops.variance_head(h.to(DEV), w.to(DEV), b.to(DEV), lens.to(DEV), c, None, bins, _index_emb(7).to(DEV),
                                torch.zeros(B, Lm, 4, device=DEV)).cpu().double()
        c64 = float(torch.tensor(c, dtype=torch.float32))
        want = (h.double() @ w.double() + b.double()) * c64
        bar = gamma(head_depth(C)) * ((h.double() * w.double()).abs().sum(-1) + b.double().abs()) * abs(c64)
        assert torch.equal(got[pad], torch.zeros_like(got[pad])), c
        err = (got - want).abs()[~pad]
        assert (err <= bar[~pad]).all(), (c, (err / bar[~pad]).max().item())
        worst = max(worst, (err / bar[~pad]).max().item())
    # without bins: the duration head, no control
    got = ops.variance_head(h.to(DEV), w.to(DEV), b.to(DEV), lens.to(DEV)).cpu().double()
    want = h.double() @ w.double() + b.double()
    bar = gamma(head_depth(C) - 1) * ((h.double() * w.double()).abs().sum(-1) + b.double().abs())
    assert ((got - want).abs()[~pad] <= bar[~pad]).all()
    parity_log(f"variance_head_pred_C{C}_scale{scale}", worst_fraction_of_bar=worst)


# ------------------------------------------------------------------------------------------------------------ variance head: buckets
def _keys_as_rows(keys, C):
    """h rows whose prediction h . e0 + 0 is the key itself (NaN and +-inf included)."""
    h = torch.zeros(1, keys.numel(), C)
    h[0, :, 0] = keys
    w = torch.zeros(C)
    w[0] = 1.0
    return h, w


@pytest.mark.parametrize("C", [4, 256])
@pytest.mark.parametrize("bins_name", list(BINS))
def test_variance_head_bucket_is_torch_bucketize(bins_name, C):
    """The bucket of every key is torch.bucketize(key, bins) of the kernel's own fp32 key, read back through emb[i] = i on a zero x:
    prediction path under scalar controls 1, 0, -1, inf and NaN (pred_out is then fp32(pred * c) exactly), and target path.  NaN keys
    (NaN prediction, inf * 0, NaN control or target) go to bucket n_edges, as ATen's search puts them."""
    bins = BINS[bins_name]
    keys = bucket_keys(bins)
    n, E = keys.numel(), bins.numel()
    h, w = _keys_as_rows(keys, C)
    b = torch.zeros(1)
    emb = _index_emb(E)
    hd, wd, bd, bins_d, emb_d = h.to(DEV), w.to(DEV), b.to(DEV), bins.to(DEV), emb.to(DEV)
    raw = ops.variance_head(hd, wd, bd).cpu()
    assert same(raw[0], keys + 0.0)
    for c in (1.0, 0.0, -1.0, math.inf, math.nan):
        x = torch.zeros(1, n, 4, device=DEV)
        pred = ops.variance_head(hd, wd, bd, None, c, None, bins_d, emb_d, x).cpu()
        assert same(pred, raw * c), c
        assert torch.equal(x[0, :, 0].cpu().long(), torch.bucketize(pred[0], bins)), c
    # target path: the key is the target, the prediction is returned unscaled
    tgt = keys[torch.randperm(n, generator=torch.Generator().manual_seed(5))][None]
    x = torch.zeros(1, n, 4, device=DEV)
    pred = ops.variance_head(hd, wd, bd, None, math.nan, tgt.to(DEV), bins_d, emb_d, x).cpu()
    assert same(pred, raw)
    idx = x[0, :, 0].cpu().long()
    assert torch.equal(idx, torch.bucketize(tgt[0], bins))
    assert (idx[tgt[0].isnan()] == E).all()


def test_variance_head_embedding_add_and_fp64_flips(parity_log):
    """Rows built so that the prediction lands within a few ulp of a bin edge: the bucket may differ from fp64's only where
    |pred64 - edge| is within the prediction's bar, and x += emb[i] is one fp32 add of the row the kernel's own key selects."""
    B, Lm, C, D = 4, 300, 256, 256
    bins = torch.linspace(-2.9, 11.4, 255)
    h = rnd(B, Lm, C, seed=11)
    w = rnd(C, seed=12, scale=0.1)
    w[0] = 0.5
    b = torch.tensor([0.3])
    c = 1.3
    c32 = float(torch.tensor(c, dtype=torch.float32))
    # half the rows: solve for h[..., 0] so that (h . w + b) * c hits an edge in fp64, then round h to fp32
    edge = bins[torch.randint(0, 255, (B, Lm // 2), generator=torch.Generator().manual_seed(13))].double()
    rest = h[:, :Lm // 2, 1:].double() @ w[1:].double() + 0.3
    h[:, :Lm // 2, 0] = ((edge / c32 - rest) / 0.5).float()
    emb = rnd(256, D, seed=14)
    x = rnd(B, Lm, D, seed=15)
    xd = x.clone().to(DEV)
    pred = ops.variance_head(h.to(DEV), w.to(DEV), b.to(DEV), None, c, None, bins.to(DEV), emb.to(DEV), xd).cpu()
    idx = torch.bucketize(pred, bins)
    assert torch.equal(xd.cpu(), x + emb[idx])
    pred64 = (h.double() @ w.double() + b.double()) * c32
    bar = gamma(head_depth(C)) * ((h.double() * w.double()).abs().sum(-1) + 0.3) * abs(c32)
    assert ((pred.double() - pred64).abs() <= bar).all()
    flips = idx != torch.bucketize(pred64, bins.double())
    margin = (pred64[..., None] - bins.double()).abs().min(-1).values
    assert (margin[flips] <= bar[flips]).all()
    parity_log("variance_head_bucket_flips_vs_fp64", flips=int(flips.sum()), rows_on_edges=B * Lm // 2)


# ------------------------------------------------------------------------------------------------------------ durations
def durations_fp64(s, c):
    """(want, lo, hi, ambiguous) for d = clamp(round(exp(s) - 1) * c, min=0) in fp64, rounded to fp32 once (the kernel's one rounding
    of the product).  expf is within 2 ulp of exp(s) (CUDA C Programming Guide, mathematical functions) and `- 1.f` rounds once more,
    so rintf may pick the other neighbour where exp(s) - 1 lies within 2 ulp(exp(s)) + 0.5 ulp(exp(s) - 1) of a half-integer: there
    either clamp(floor * c) or clamp((floor + 1) * c) is accepted.  exp(s) past fp32's range is inf, as expf returns."""
    s64, c64 = s.double(), torch.as_tensor(c, dtype=torch.float32).double()
    ex = torch.exp(s64)
    ex = torch.where(ex > FLT_MAX, torch.full_like(ex, math.inf), ex)
    e = ex - 1
    fin = torch.isfinite(e)
    win = torch.where(fin, 2 * ulp32(torch.where(fin, ex, 0)) + 0.5 * ulp32(torch.where(fin, e, 0)), 0)
    lo = torch.floor(e)
    amb = fin & ((e - lo - 0.5).abs() <= win)
    f = lambda r: torch.clamp(r * c64, min=0).float()
    return f(torch.round(e)), f(lo), f(lo + 1), amb


def check_durations(d, s, c, valid=None):
    """d_rounded (the kernel's) against fp64; returns the number of accepted near-tie cases."""
    want, lo, hi, amb = durations_fp64(s, c)
    if valid is not None:
        want = torch.where(valid, want, 0.0)
        amb = amb & valid
    ok = (d.isnan() & want.isnan()) | (d == want) | (amb & ((d == lo) | (d == hi)))
    bad = [tuple(i) for i in ok.logical_not().nonzero().tolist()[:5]]
    assert ok.all(), [(i, float(s[i]), float(d[i]), float(want[i])) for i in bad]
    return int((amb & (d != want)).sum())


def expected_frames(d, valid=None):
    """reps = max(trunc(d), 0), wild (NaN, +-inf, > 1e6: the reference's int() raises or it would size a gigantic output) -> 0."""
    wild = ~((d <= 1e6) & (d > -math.inf))
    if valid is not None:
        wild = wild & valid
    reps = torch.where(wild, 0.0, d.nan_to_num()).trunc().clamp(min=0).long()
    if valid is not None:
        reps = torch.where(valid, reps, 0)
    return reps.cumsum(1), int(wild.sum())


def check_counts(cum, mel_lens, mel_lens32, stats, d, valid=None):
    want_cum, wild = expected_frames(d, valid)
    total = want_cum[:, -1]
    if cum is not None:
        assert torch.equal(cum.long(), want_cum)
    assert torch.equal(mel_lens.long(), total) and (mel_lens32 is None or torch.equal(mel_lens32.long(), total))
    assert stats.tolist() == [int(total.max()), int(total.sum()), wild]
    return wild


def duration_logits(B, Lm, seed):
    """Random log-durations, one all-zero utterance (d = 0 everywhere), half-integer ties round(k + 0.5) for even and odd k, and
    s = +-inf, NaN, 89 (expf overflows) and 14 (> 1e6 frames)."""
    s = rnd(B, Lm, seed=seed, scale=1.0) + 1.0
    if B > 1:
        s[1] = 0.0
    ties = torch.log(torch.arange(8, dtype=torch.float64) + 1.5).float()
    special = torch.tensor([math.inf, -math.inf, math.nan, 89.0, 14.0, -30.0])
    row = torch.cat([ties, special])[:Lm]
    s[0, -row.numel():] = row
    return s


@pytest.mark.parametrize("d_control", [1.0, 2.5, 0.0, -1.0, math.inf, math.nan])
@pytest.mark.parametrize("Lm", [1, 31, 255, 256, 257, 1000])
def test_durations_against_fp64(Lm, d_control, parity_log):
    """Predicted durations, scalar d_control: d_rounded per durations_fp64, cum / mel_lens / mel_lens32 as int64 prefix sums of the
    kernel's own d, len_stats = [max, sum, wild count] exactly.  L crosses the 256-thread block scan's carry at several offsets."""
    B = 4
    s = duration_logits(B, Lm, seed=Lm)
    d, cum, mel_lens, mel_lens32, stats = ops.durations(s.to(DEV), False, d_control)
    d = d.cpu()
    near = check_durations(d, s, d_control)
    wild = check_counts(cum.cpu(), mel_lens.cpu(), mel_lens32.cpu(), stats.cpu(), d)
    if Lm >= 14:
        assert wild >= 1                                        # s = NaN at least
    parity_log(f"durations_L{Lm}_c{d_control}", near_tie_cases=near, wild=wild)


def test_teacher_forced_durations_truncate_and_count_wild():
    """use_target: reps = max(trunc(d), 0); NaN, +-inf and 1e6 + 1 are wild (0 frames, counted)."""
    t = torch.tensor([[2.7, -2.7, 0.5, -0.0, 0.0, math.nan, 7.0, math.inf, -math.inf, 1e6, 1e6 + 1, 3.99]])
    t = torch.cat([t, torch.flip(t, [1]), torch.full_like(t, 1.5)])
    d, cum, mel_lens, mel_lens32, stats = ops.durations(t.to(DEV), True, math.nan)
    assert d is None
    assert check_counts(cum.cpu(), mel_lens.cpu(), mel_lens32.cpu(), stats.cpu(), t) == 8
    assert cum[0].tolist() == [2, 2, 2, 2, 2, 2, 9, 9, 9, 1000009, 1000009, 1000012]


# ------------------------------------------------------------------------------------------------------------ length regulator
@pytest.mark.parametrize("with_pos", [False, True])
def test_length_regulate_is_a_gather(with_pos):
    """y[b, t] = x[b, i(t)] (+ pos[t]) for t < min(total_b, T), pos[t] or 0 after: the reference's repeat_interleave and pad(max_len),
    which truncates when T is below the total.  Zero durations at the first and last phoneme and in runs; L = 1."""
    D = 256
    for reps in ([[0, 2, 0, 0, 3, 1, 0, 4, 0], [3, 0, 0, 0, 0, 0, 0, 0, 2], [0, 0, 0, 0, 0, 0, 0, 0, 7]], [[5]], [[0], [3]]):
        reps = torch.tensor(reps)
        B, Lm = reps.shape
        cum = reps.cumsum(1).to(torch.int32)
        x = rnd(B, Lm, D, seed=Lm)
        tot = reps.sum(1)
        pos = rnd(int(tot.max()) + 8, D, seed=3)
        for T in sorted({1, max(int(tot.min()) - 1, 1), int(tot.max()) - 1, int(tot.max()), int(tot.max()) + 5} - {0}):
            want = torch.zeros(B, T, D)
            for b in range(B):
                e = torch.repeat_interleave(x[b], reps[b], dim=0)[:T]
                want[b, :e.shape[0]] = e
            if with_pos:
                want = want + pos[:T]
            got = ops.length_regulate(x.to(DEV), cum.to(DEV), T, pos.to(DEV) if with_pos else None)
            assert torch.equal(got.cpu(), want), (reps.tolist(), T)


# ------------------------------------------------------------------------------------------------------------ through the model
def _lj_model(lj_configs, seed):
    sd = synth.fastspeech2_state_dict(*lj_configs, seed=seed)
    m = FastSpeech2(*lj_configs)
    m.load_state_dict(sd)
    return m.to(DEV).eval(), sd


SPECIAL_CONTROLS = {(0, 1): 0.0, (0, 2): -1.0, (0, 3): math.inf, (0, 4): math.nan, (2, 0): math.inf, (3, 5): math.nan}


@pytest.mark.parametrize("ragged", [False, True])
def test_per_phoneme_d_control_durations_against_fp64(ragged, lj_configs):
    """The per-element control instantiation of durations_kernel (padded and ragged) through fs2_acoustic_encode_ctl: d_rounded against
    fp64 of the kernel's own log-durations, mel_lens and len_stats from its own d.  Ragged: columns past src_lens[b] are 0 and not
    counted; padded: they are the reference's clamp(round(exp(0) - 1) * c) (NaN for a NaN or inf control there)."""
    m, _ = _lj_model(lj_configs, seed=101)
    spk, texts, lens, Lm = synth.make_batch(4, 40, seed=102, min_len=9)
    c = 0.5 + 1.5 * torch.rand(4, Lm, generator=torch.Generator().manual_seed(103))
    for (b, l), v in SPECIAL_CONTROLS.items():
        c[b, l] = v
    c[1, -1] = math.nan                                          # past src_lens[1] (make_batch keeps utterance 1 shorter than Lm)
    assert int(lens[1]) < Lm
    out = m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm, max_mel_len=64, d_control=c.to(DEV), ragged=ragged)
    torch.cuda.synchronize()
    stats = m._stats_host.clone()
    logd, d = out[4].cpu(), out[5].cpu()
    valid = torch.arange(Lm)[None, :] < lens[:, None] if ragged else None
    if ragged:
        assert torch.equal(d[~valid], torch.zeros_like(d[~valid]))
    check_durations(d, logd, c, valid)
    wild = check_counts(None, out[9].cpu(), None, stats, d, valid)
    assert wild >= 3


@pytest.mark.parametrize("ragged", [False, True])
def test_nan_d_control_raises(ragged, lj_configs):
    """A NaN duration control on a valid phoneme makes the duration NaN, and the reference's int() raises on it: so does forward."""
    m, _ = _lj_model(lj_configs, seed=104)
    spk, texts, lens, Lm = synth.make_batch(3, 24, seed=105, min_len=9)
    c = torch.ones(3, Lm)
    c[1, 2] = math.nan
    with pytest.raises(L.Fs2Error, match="NaN"):
        m(spk.to(DEV), texts.to(DEV), lens.to(DEV), Lm, d_control=c.to(DEV), ragged=ragged)


def test_nan_and_inf_p_control_against_the_oracle(lj_configs, parity_log):
    """A per-phoneme p_control with NaN, +inf and -inf elements: pitch predictions are fp32(pred * c) bit for bit, NaN ones take bucket
    n_edges and +-inf the outer buckets, as torch.bucketize does in the oracle, so the mel equals the oracle's.  Durations are the
    oracle's own (teacher-forced), so only the pitch / energy decisions are under test."""
    m, sd = _lj_model(lj_configs, seed=106)
    spk, texts, lens, Lm = synth.make_batch(2, 24, seed=107, min_len=12)
    p = torch.ones(2, Lm)
    p[0, 3], p[0, 7], p[0, 9], p[1, 5] = math.nan, math.inf, -math.inf, math.nan
    free = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
    tf = (None, free[9], int(free[9].max()), None, None, free[5].long())
    ref = O.fastspeech2_forward(sd, spk, texts, lens, Lm, *tf, p_control=p)
    dev = lambda xs: [v.to(DEV) if torch.is_tensor(v) else v for v in xs]
    out = m(*dev((spk, texts, lens, Lm) + tf), p_control=p.to(DEV))
    plain = m(*dev((spk, texts, lens, Lm) + tf))
    assert same(out[2].cpu(), plain[2].cpu() * p)
    for i, nm in ((2, "pitch"), (3, "energy")):
        o, r = out[i].cpu(), ref[i]
        assert torch.equal(o.isnan(), r.isnan()) and torch.equal(o.isinf(), r.isinf()), nm
        fin = torch.isfinite(r)
        assert (o[fin] - r[fin]).abs().max() < 1e-4, nm
        edges = sd[f"variance_adaptor.{nm}_bins"]
        assert torch.equal(torch.bucketize(o, edges), torch.bucketize(r, edges)), nm
    assert (torch.bucketize(out[2].cpu(), sd["variance_adaptor.pitch_bins"])[p.isnan()] == 255).all()
    e = {"mel": (out[0].cpu() - ref[0]).abs().max().item(), "postnet": (out[1].cpu() - ref[1]).abs().max().item()}
    parity_log("fs2_nan_inf_p_control_vs_oracle", **e)
    assert e["mel"] < MEL_TOL and e["postnet"] < MEL_TOL, e


# ------------------------------------------------------------------------------------------------------------ conv_post
def conv_post_depth(kernel, C, taps):
    """Rounding depth n of each conv_post kernel's sum  bias + sum_{j,c} w[j][c] * lrelu(x):
      - c32 (register-resident, C = 32, k = 7): each of the 8 lanes of a row group owns 4 channels and folds a row into an output's
        sliding accumulator with a chain of 4 FMAs; an output receives its 7 rows in order, so its lane partial passes 7 * 4 = 28 FMAs,
        then the 3-shuffle reduction over the 8 lanes (3) and the bias add (1): n = 32;
      - staged (shared memory, any C % 4 == 0): acc starts at the bias and takes taps * C FMAs in order: n = taps * C.
    lrelu is computed in fp32 exactly as the kernel does (one multiply by the fp32 slope) and the sum in fp64 from there, so
    |acc - acc64| <= gamma_n (|b| + sum |w * lrelu(x)|)."""
    return 32 if kernel == "c32" else taps * C


CONV_POST_KERNELS = {"c32": (32, 7, True), "staged_unaligned_c32": (32, 7, False), "staged_c16_k5": (16, 5, True),
                     "staged_c8_k7": (8, 7, True)}


@pytest.mark.parametrize("ragged", [False, True])
@pytest.mark.parametrize("T", [119, 120, 121, 255, 256, 257, 12345])
@pytest.mark.parametrize("kernel", list(CONV_POST_KERNELS))
def test_conv_post_against_fp64(kernel, T, ragged, parity_log):
    """wav = tanh(acc) per element within gamma_n S (1 - tanh(|acc64| - gamma_n S)^2) + 2 ulp(y), S = |b| + sum |w * lrelu(x)|, n per
    conv_post_depth: the first term carries the sum's error through tanh's slope, the second is tanhf's own error (2 ulp, CUDA C
    Programming Guide).  Activations are 2^e * N(0, 1) with e from [-12, 6] per block of 16 rows, so outputs run from tanh's linear range to
    saturation.  T around the c32 kernel's 120-row groups and the staged kernel's 256-row tiles; the unaligned case passes x at a 4-byte
    offset, which sends C = 32, k = 7 to the staged kernel.  Ragged: lens with lens_scale 256, rows past lens[b] * 256 read as zero and
    wav there exactly 0."""
    C, k, aligned = CONV_POST_KERNELS[kernel]
    B = 3
    g = torch.Generator().manual_seed(T * 7 + C)
    blk = torch.arange(B)[:, None] * 3 + torch.arange(T)[None, :] // 16          # 16-row blocks visit every exponent in [-12, 6]
    x = torch.randn(B, T, C, generator=g) * torch.exp2((blk * 7 % 19 - 12).float())[..., None]
    w = torch.randn(k, C, generator=g) * 0.1
    bias = torch.tensor([2.0 ** -14])
    slope = torch.tensor(0.01, dtype=torch.float32)
    lens = torch.tensor([(T + 255) // 256, (T // 256) // 2, T // 256], dtype=torch.int32) if ragged else None
    n_b = torch.clamp(lens.long() * 256, max=T) if ragged else torch.full((B,), T)
    if aligned:
        xd = x.to(DEV)
    else:
        flat = torch.empty(B * T * C + 1, device=DEV)
        xd = flat[1:].view(B, T, C)
        xd.copy_(x.to(DEV))
        assert xd.data_ptr() % 16 != 0
    got = ops.conv_post(xd, w.to(DEV), bias.to(DEV), float(slope), None if lens is None else lens.to(DEV), 256).cpu().double()
    xa = torch.where(x > 0, x, x * slope)
    live = torch.arange(T)[None, :] < n_b[:, None]
    xa = xa * live[..., None]
    conv = lambda a, ww: torch.nn.functional.conv1d(a.transpose(1, 2), ww.t()[None], padding=(k - 1) // 2)[:, 0]
    acc64 = conv(xa.double(), w.double()) + float(bias)
    S = conv(xa.double().abs(), w.double().abs()) + abs(float(bias))
    dacc = gamma(conv_post_depth(kernel.split("_")[0], C, k)) * S
    y64 = torch.tanh(acc64)
    bar = dacc * (1 - torch.tanh((acc64.abs() - dacc).clamp(min=0)) ** 2) + 2 * ulp32(y64)
    assert torch.equal(got[~live], torch.zeros_like(got[~live]))
    err = (got - y64).abs()[live]
    frac = (err / bar[live]).max().item()
    assert frac <= 1.0, (kernel, T, frac)
    assert (y64.abs() > 0.999)[live].any() and (y64.abs() < 1e-2)[live].any()      # both tanh regimes are covered
    parity_log(f"conv_post_{kernel}_T{T}_{'ragged' if ragged else 'padded'}", worst_fraction_of_bar=frac)
