"""CPU: the op decomposition the CUDA path executes (packing + model.cu's launch sequence, emulated op by op from the
C-ABI contracts) reproduces the oracle.  Tolerances: fp32 re-association only (no reduced precision anywhere)."""
import torch

from fastspeech2_b200 import configs, packing, synth
from oracle import fs2_oracle as O
from tests import emul_cabi as E

CFG = dict(n_head=2, k1=9, k2=1, n_enc=4, n_dec=6, vp_kernel=3, n_postnet=5, post_k=5)


def _pk(sd, multi):
    return packing.pack_acoustic(lambda k: sd[k], 4, 6, 5, multi)


def test_acoustic_free_running_lj(lj_configs):
    pc, mc = lj_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=3)
    spk, texts, lens, L = synth.make_batch(3, 28, seed=5, min_len=9)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, L, p_control=1.2, d_control=0.9)
    mel, post, p, e, logd, d, mel_len = E.acoustic_forward(_pk(sd, False), CFG, spk, texts, lens, p_control=1.2, d_control=0.9)
    assert torch.equal(mel_len, ref[9]) and torch.equal(d, ref[5])
    for got, want, tol in ((mel, ref[0], 2e-5), (post, ref[1], 2e-5), (p, ref[2], 5e-6), (e, ref[3], 5e-6), (logd, ref[4], 5e-6)):
        assert (got - want).abs().max() < tol


def test_acoustic_teacher_forced_libri(libri_configs):
    pc, mc = libri_configs
    sd = synth.fastspeech2_state_dict(pc, mc, seed=4)
    spk, texts, lens, L = synth.make_batch(2, 20, seed=6, n_speakers=904, min_len=11)
    g = torch.Generator().manual_seed(1)
    d_t = torch.randint(0, 6, (2, L), generator=g) * (torch.arange(L)[None] < lens[:, None])
    p_t = torch.randn(2, L, generator=g) * 2
    e_t = torch.randn(2, L, generator=g) * 2
    mel_lens = d_t.sum(1)
    T = int(mel_lens.max()) + 3
    ref = O.fastspeech2_forward(sd, spk, texts, lens, L, None, mel_lens, T, p_t, e_t, d_t)
    mel, post, p, e, logd, d, mel_len = E.acoustic_forward(_pk(sd, True), CFG, spk, texts, lens, p_target=p_t, e_target=e_t,
                                                          d_target=d_t.float(), mel_lens=mel_lens, max_mel_len=T)
    assert torch.equal(mel_len, ref[9])
    for got, want in ((mel, ref[0]), (post, ref[1]), (p, ref[2]), (e, ref[3]), (logd, ref[4])):
        assert (got - want).abs().max() < 2e-5


def test_acoustic_frame_level_variances(scratch):
    """config/LJSpeech_paper style: pitch / energy predicted per mel frame after the length regulator (modules.py:139-148)."""
    import copy
    pc, mc = configs.make_configs("LJSpeech", scratch)
    pc = copy.deepcopy(pc)
    pc["preprocessing"]["pitch"]["feature"] = "frame_level"
    pc["preprocessing"]["energy"]["feature"] = "frame_level"
    sd = synth.fastspeech2_state_dict(pc, mc, seed=8)
    spk, texts, lens, L = synth.make_batch(2, 18, seed=9, min_len=11)
    ref = O.fastspeech2_forward(sd, spk, texts, lens, L, p_control=0.9, pitch_level="frame_level", energy_level="frame_level")
    mel, post, p, e, logd, d, mel_len = E.acoustic_forward(_pk(sd, False), CFG, spk, texts, lens, p_control=0.9, pitch_frame=True,
                                                          energy_frame=True)
    assert torch.equal(mel_len, ref[9]) and p.shape == ref[2].shape == mel.shape[:2]
    for got, want in ((mel, ref[0]), (post, ref[1]), (p, ref[2]), (e, ref[3]), (logd, ref[4])):
        assert (got - want).abs().max() < 2e-5


def test_vocoder_decomposition():
    h = configs.HIFIGAN_CONFIG
    sd = synth.hifigan_state_dict(h, seed=2)
    mel = synth.make_mel(2, 12, seed=1)
    want = O.hifigan_forward(sd, mel)
    folded = O.fold_weight_norm(sd)
    pk = packing.pack_vocoder(lambda b: folded[b + ".weight"], lambda b: folded[b + ".bias"], h["upsample_rates"], 12, 3)
    got = E.vocoder_forward(pk, h["upsample_rates"], h["resblock_kernel_sizes"], h["resblock_dilation_sizes"],
                            mel.transpose(1, 2).contiguous())
    assert got.shape == (2, 12 * 256)
    assert (got - want[:, 0]).abs().max() < 2e-5


def test_resblock_unfused_bar_rejects_a_single_pass_fp16_tile():
    """The GPU test of the fused ResBlock kernel (test_gpu_ops.test_resstack_fused) bounds its difference from the same group built from
    per-layer tensor-core convs by RESSTACK_UNFUSED_C 2^-24 S per element, S carried through the group (E.resstack_contract).  Evaluated
    in fp64 on the kernels' rounded operands, the group with the E4M3 correction dropped (single-pass fp16) differs from the f16 + f8
    contract in every 128-row block of every case by more than 10x that bar, so a kernel that lost the correction in any one of its
    (longer) tiles fails that test."""
    import functools
    from tests import test_gpu_ops as G
    from tests.test_gpu_tc_precision import RESSTACK_UNFUSED_C
    for case in G.RESSTACK_CASES:
        B, N, C, ks, ds = case
        x, w1, b1, w2, b2 = G._resstack_case(case)
        full = E.resblock_group(x, ks, ds, w1, b1, w2, b2, conv=E.conv1d_f8)
        fp16 = E.resblock_group(x, ks, ds, w1, b1, w2, b2, conv=functools.partial(E.conv1d_f8, fp16_only=True))
        _, S, _ = E.resstack_contract(x, ks, ds, w1, b1, w2, b2)
        diff = (full - fp16).abs() / (E.U24 * S)
        blocks = [diff[b, s:s + 128].max().item() for b in range(B) for s in range(0, N, 128) if min(N - s, 128) >= 32]
        if blocks:
            assert min(blocks) > 10 * RESSTACK_UNFUSED_C, (case, min(blocks))


def test_split_conv_transpose_matches_torch():
    g = torch.Generator().manual_seed(0)
    for u, cin, cout in ((8, 16, 8), (2, 8, 4)):
        w = torch.randn(cin, cout, 2 * u, generator=g)
        x = torch.randn(2, 9, cin, generator=g)
        want = torch.nn.functional.conv_transpose1d(x.transpose(1, 2), w, stride=u, padding=u // 2).transpose(1, 2)
        wa, wb = packing.split_conv_transpose(w, u)
        ya = E.conv1d(x, wa, None, pad_left=1)
        yb = E.conv1d(x, wb, None, pad_left=0)
        got = torch.cat([ya, yb], -1).reshape(2, 9 * u, cout)
        assert (got - want).abs().max() < 1e-5


def test_conv_post_sliding_window_schedule():
    """The work decomposition of conv_post_c32_kernel (rowwise.cu), emulated lane for lane: 8 lanes per time row (4 channels each), groups
    of 18 x 7 input rows = 120 output rows + a 6-row halo, 7 sliding accumulators per lane (accumulator k of row r belongs to output
    r - 3 + k and takes tap 6 - k), an 8-lane sum when an output has seen its last row, stores in runs of 8 samples.  Must equal
    lrelu -> Conv1d(32, 1, 7, padding=3) -> tanh (hifigan/models.py:161-163) for lengths around the group and store-run boundaries,
    with every sample written exactly once."""
    import numpy as np
    TAPS, PAD, BLOCKS = 7, 3, 18
    ROWS = BLOCKS * TAPS - 2 * PAD
    rng = np.random.default_rng(0)
    for T in (1, 5, 7, 8, 9, 119, 120, 121, 127, 128, 250, 963):
        x = rng.standard_normal((T, 32))
        w = rng.standard_normal((TAPS, 32)) * 0.1
        xa = np.where(x > 0, x, 0.01 * x)
        want = np.array([np.tanh(0.05 + sum((xa[t + j - PAD] * w[j]).sum() for j in range(TAPS) if 0 <= t + j - PAD < T)) for t in range(T)])
        out = np.full(T, np.nan)
        for g in range((T + ROWS - 1) // ROWS):
            t0 = g * ROWS
            tend = min(t0 + ROWS, T)
            s, keep = np.zeros((8, TAPS)), np.zeros(8)
            for blk in range(BLOCKS):
                for i in range(TAPS):
                    r = t0 - PAD + blk * TAPS + i
                    v = xa[r].reshape(8, 4) if 0 <= r < T else np.zeros((8, 4))
                    for k in range(TAPS):
                        s[:, k] += (v * w[TAPS - 1 - k].reshape(8, 4)).sum(1)
                    tot = s[:, 0].sum()
                    s[:, :-1] = s[:, 1:].copy()
                    s[:, -1] = 0.0
                    t = r - PAD
                    if t0 <= t < tend:
                        o = (t - t0) & 7
                        keep[o] = tot
                        if o == 7 or t == tend - 1:
                            for sub in range(o + 1):
                                assert np.isnan(out[t - o + sub])
                                out[t - o + sub] = np.tanh(keep[sub] + 0.05)
        assert not np.isnan(out).any() and np.abs(out - want).max() < 1e-12, T


# The exact-kernel bars of tests/test_gpu_ops.py against the faults they are there to catch, emulated in fp64 on the same cases: each
# must put some element at least 100x past its bar, so a kernel with that fault fails its test.
REJECT = 100.0


def test_exact_conv_bar_rejects_a_dropped_k_step():
    """One 16-channel K-step left out, at the longest sum of test_conv1d's table (K = 9216): every 64-row tile is caught."""
    from tests import test_gpu_ops as G
    case = max((G._case_opts(c)[0] for c in G.CONV_CASES), key=lambda c: c[2] * c[4])
    assert case[2] * case[4] == 9216
    B, T, Cin, N, taps, dil, pad, in_act, out_act, _, alpha, _, _ = case
    x, w, bias, res, y0, lens = G._conv_case(case)
    want = E.conv1d(x.double(), w.double(), bias.double(), dil, pad, in_act, 0.1, out_act, 0.1)
    scale = G.conv_scale(x, w, bias, dil, pad, in_act, 0.1, None, alpha, None, None)
    wf = w.clone()
    wf[taps // 2, 7 * 16:8 * 16] = 0.0
    fault = E.conv1d(x.double(), wf.double(), bias.double(), dil, pad, in_act, 0.1, out_act, 0.1)
    bm = G.simt_plan(B, T, Cin, N, taps)[0]
    tiles = [G.normalised_err(fault[b:b + 1, s:s + bm], want[b:b + 1, s:s + bm], scale[b:b + 1, s:s + bm]) for b in range(B) for s in range(0, T, bm)]
    assert min(tiles) > REJECT * G.CONV_EXACT_C, (min(tiles), G.CONV_EXACT_C)


def test_exact_conv_bar_rejects_a_halo_row_off_by_one():
    """The first row of the second 64-row tile reading its first tap's input one row late (a halo load off by one at a tile edge)."""
    from tests import test_gpu_ops as G
    case, opts = next(G._case_opts(c) for c in G.CONV_CASES if G._case_opts(c)[0][:5] == (2, 300, 64, 48, 5))
    B, T, Cin, N, taps, dil, pad, in_act, out_act, _, alpha, _, _ = case
    slope = opts.get("in_slope", 0.1)
    x, w, bias, _, _, _ = G._conv_case(case)
    bm = G.simt_plan(B, T, Cin, N, taps)[0]
    t, shift = bm, -pad
    xd, wd = x.double(), w.double()
    acc = E.conv1d(xd, wd, None, dil, pad, in_act, slope)
    want = E.conv1d_epilogue(acc, bias.double(), out_act, 0.1)
    xa = E._act(xd, in_act, slope)
    acc[:, t] += (xa[:, t + shift + 1] - xa[:, t + shift]) @ wd[0]
    fault = E.conv1d_epilogue(acc, bias.double(), out_act, 0.1)
    scale = G.conv_scale(x, w, bias, dil, pad, in_act, slope, None, alpha, None, None)
    for b in range(B):
        e = G.normalised_err(fault[b:b + 1, t:t + 1], want[b:b + 1, t:t + 1], scale[b:b + 1, t:t + 1])
        assert e > REJECT * G.CONV_EXACT_C, (b, e)


def _tiled_softmax_attention(qkv, lens, rescale=True, mask_before_max=True):
    """The exact attention kernel's online softmax over 64-key tiles in fp64, with p = exp(s - m) rounded through fp32 as the kernel
    computes it.  rescale=False: O and l are not rescaled when a later tile raises the running max.  mask_before_max=False: the max
    is taken over every key of the visited tiles, the masked ones past n in the last tile included."""
    B, T, _ = qkv.shape
    q, k, v = (qkv[..., i * 256:(i + 1) * 256].double().reshape(B, T, 2, 128).permute(0, 2, 1, 3) for i in range(3))
    out = torch.zeros(B, 2, T, 128, dtype=torch.float64)
    for b, n in enumerate(lens):
        n = min(max(n, 0), T)
        if n == 0:
            continue
        s = q[b] @ k[b].transpose(-1, -2) / 128 ** 0.5
        key = torch.arange(T)
        m = torch.full((2, T, 1), float("-inf"), dtype=torch.float64)
        l = torch.zeros(2, T, 1, dtype=torch.float64)
        o = torch.zeros(2, T, 128, dtype=torch.float64)
        for k0 in range(0, n, 64):
            st = s[:, :, k0:k0 + 64]
            valid = key[k0:k0 + 64] < n
            m_tile = (st if not mask_before_max else st.masked_fill(~valid, float("-inf"))).amax(-1, keepdim=True)
            m_new = torch.maximum(m, m_tile)
            p = torch.exp((st - m_new).float()).double().masked_fill(~valid, 0.0)
            c = torch.exp(m - m_new) if rescale else torch.ones_like(m)
            l = l * c + p.sum(-1, keepdim=True)
            o = o * c + p @ v[b][:, k0:k0 + 64]
            m = m_new
        out[b] = o / l
        out[b, :, n:] = 0.0
    return out.permute(0, 2, 1, 3).reshape(B, T, 256)


def test_attention_bar_rejects_a_missing_rescale_and_a_max_over_masked_keys():
    """On test_attention_adversarial_scores' cases: the emulated kernel matches fp64 within the bar as it is; without the online
    rescale (row max in the last key tile) or with masked keys in the max (they hold the largest scores), every utterance with more
    than one key tile, respectively with masked keys in its last tile, is caught."""
    from tests import test_gpu_ops as G
    bar = max(G.ATT_EXACT_C.values())
    for kind, fault in (("last_tile_max", dict(rescale=False)), ("masked_max", dict(mask_before_max=False))):
        T, lens = next((T, lens) for k, T, lens in G.ATT_ADV_CASES if k == kind)
        qkv = G.attention_qkv(kind, lens, T)
        kl = torch.tensor(lens, dtype=torch.int32)
        want = E.attention(qkv.double(), 2, kl)
        scale = G.attention_bar_scale(qkv, kl)
        good = _tiled_softmax_attention(qkv, lens)
        bad = _tiled_softmax_attention(qkv, lens, **fault)
        for b, n in enumerate(lens):
            n = min(max(n, 0), T)
            e_good = G.attention_normalised_err(good[b:b + 1], want[b:b + 1], scale[b:b + 1])
            assert e_good < bar / 4, (kind, b, e_good)
            if (kind == "last_tile_max" and n > 64) or (kind == "masked_max" and 0 < n < T and n % 64):
                e = G.attention_normalised_err(bad[b:b + 1], want[b:b + 1], scale[b:b + 1])
                assert e > REJECT * bar, (kind, b, n, e)


def test_layernorm_bar_rejects_a_one_pass_variance():
    """E[x^2] - E[x]^2 in fp32 on test_layernorm's rows with |mean| / std up to 1e4."""
    from tests import test_gpu_ops as G
    for C in (80, 256, 1024):
        x = G.layernorm_rows(C)
        gm, bt = 1 + G.rnd(C, seed=2, scale=0.1), G.rnd(C, seed=3, scale=0.1)
        want = E.layernorm(x.double(), gm.double(), bt.double())
        mean = x.mean(-1, keepdim=True)
        var = ((x * x).mean(-1, keepdim=True) - mean * mean).clamp_min(0.0)
        fault = (x - mean) * torch.rsqrt(var + 1e-5) * gm + bt
        e = G.normalised_err(fault, want, G.ln_scale(x, gm, bt))
        assert e > REJECT * G.LN_C, (C, e)
