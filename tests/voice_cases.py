"""Eight FastSpeech2 voices that differ wherever a voice can differ, and the batches that drive the acoustic voices mode into the plans
large batches pick (TEST INFRASTRUCTURE, shared by tests/test_acoustic_voices_plans_cpu.py and tests/test_gpu_acoustic_voices_plans.py).

In the voices mode (VoiceBank, fs2_acoustic_{encode,decode}_voices) every work item reads its weights, weight-scale headers, bias and
tables from its own utterance's voice.  A test can only see a voice mix-up where the voices differ, so the voices here are built to
differ in what the kernels read per voice, not only in their random draws:
  * weight scales: every tensor-core layer's packed header (packing.pack_conv_tc's 1 / scale, the power of two that puts max|w| in
    [8192, 16384)) differs between every pair of voices, and every K-segmented conv (encoder FFT blocks, variance predictors:
    packing.pack_conv_tc_segments, one header per (tap, 256-channel) segment) has at least two distinct segment headers within a
    voice, in a pattern that changes from voice to voice.  Synthetic seeds alone give every voice, and every segment of a conv, the
    same header.  The rescaling is by powers of two, compensated where the model is homogeneous: an FFN's hidden channel c by 2^a_c in
    w_1 and 2^-a_c in w_2 (ReLU), the value projection against the attention's output projection, mel_linear against the decoder's
    last LayerNorm.  Elsewhere (query / key scale, per-tap scales, the predictors, the PostNet's folded BatchNorm) the next LayerNorm
    or tanh takes the scale and the voice is a slightly different, still sane model;
  * tables: each voice has its own position tables (within max_seq_len), duration-head bias and pitch / energy bins.
check_voices asserts both on the CPU; check_sane runs every voice through the CPU oracle."""
import math

import torch

from fastspeech2_b200 import _lib as L, packing, synth
from tests import conv_group_cases as G

MAX_VOICES = 8
SEEDS = tuple(71 + v for v in range(MAX_VOICES))
# keys of the state dict no kernel reads (BatchNorm's step counter)
UNREAD = ("num_batches_tracked",)


def _shift(v, j):
    """The power-of-two exponent of layer j in voice v: a permutation of -4..3 over the voices for every j, rotating with j so that no
    voice is the scaled-up one everywhere."""
    return (v + 3 * j) % MAX_VOICES - 4


def _pattern(v, n, salt):
    """n bits, not all equal, distinct for the 8 voices where n allows (2^n - 2 >= 8): the within-voice pattern of segment exponents."""
    m = (1 << n) - 2
    code = (v * 5 + salt) % m + 1
    return [(code >> k) & 1 for k in range(n)]


def _postnet_exponent(sd, i):
    """log2 of the weight-scale header of PostNet conv i as packing packs it (BatchNorm folded)."""
    p = f"postnet.convolutions.{i}"
    wf, _ = packing.fold_batchnorm(sd[p + ".0.conv.weight"], sd[p + ".0.conv.bias"], sd[p + ".1.weight"], sd[p + ".1.bias"],
                                   sd[p + ".1.running_mean"], sd[p + ".1.running_var"])
    return -int(math.log2(packing.split_fp16(wf)[2]))


def voice_state_dict(pc, mc, v, post_ref=None):
    """Voice v (0 <= v < 8): synth.fastspeech2_state_dict at SEEDS[v], rescaled and given its own tables as the module docstring says.
    post_ref: {i: the log2 header PostNet conv i is given in a voice whose shift is 0} (None: this seed's own)."""
    sd = synth.fastspeech2_state_dict(pc, mc, seed=SEEDS[v])
    tr = mc["transformer"]
    F = tr["conv_filter_size"]
    j = 0

    def nxt():
        nonlocal j
        j += 1
        return _shift(v, j)
    for side, n in (("encoder", tr["encoder_layer"]), ("decoder", tr["decoder_layer"])):
        for i in range(n):
            a, f = f"{side}.layer_stack.{i}.slf_attn.", f"{side}.layer_stack.{i}.pos_ffn."
            # attention: q, k, v by 2^h, the output projection by 2^-h (exact on the value path); for h > 0 the key by 2^-h instead,
            # so the scores keep their scale, for h < 0 the scores flatten by 4^h
            h = nxt()
            for w, e in (("w_qs", h), ("w_ks", -h if h > 0 else h), ("w_vs", h)):
                sd[a + w + ".weight"] *= 2.0 ** e
                sd[a + w + ".bias"] *= 2.0 ** e
            sd[a + "fc.weight"] *= 2.0 ** -h
            # FFN: hidden chunk k (256 channels) by 2^a_k in w_1 and 2^-a_k in w_2 (ReLU: exact).  The encoder's w_2 is K-segmented by
            # those chunks, so a_k varies within the voice there; its w_1 is segmented by tap, so its taps get 2^q_t on top (not exact)
            h = nxt()
            nck = F // packing.SEG_CIN
            ak = [h + p for p in _pattern(v, nck, i)] if side == "encoder" else [h] * nck
            for k, ex in enumerate(ak):
                ch = slice(k * packing.SEG_CIN, (k + 1) * packing.SEG_CIN)
                sd[f + "w_1.weight"][ch] *= 2.0 ** ex
                sd[f + "w_1.bias"][ch] *= 2.0 ** ex
                sd[f + "w_2.weight"][:, ch] *= 2.0 ** -ex
            if side == "encoder":
                k1 = sd[f + "w_1.weight"].shape[2]
                for t, q in enumerate(_pattern(v, k1, 3 * i + 1)):
                    sd[f + "w_1.weight"][:, :, t] *= 2.0 ** q
    for nm in ("duration", "pitch", "energy"):
        for c in (1, 2):
            # predictor convs (K-segmented by tap): tap t by 2^(h + p_t), the bias by 2^h; the ReLU + LayerNorm after takes 2^h
            p = f"variance_adaptor.{nm}_predictor.conv_layer.conv1d_{c}.conv."
            h = nxt()
            for t, q in enumerate(_pattern(v, sd[p + "weight"].shape[2], 2 * j)):
                sd[p + "weight"][:, :, t] *= 2.0 ** (h + q)
            sd[p + "bias"] *= 2.0 ** h
    # mel_linear by 2^h against the decoder's last LayerNorm by 2^-h (exact)
    h = nxt()
    sd["mel_linear.weight"] *= 2.0 ** h
    last = f"decoder.layer_stack.{tr['decoder_layer'] - 1}.pos_ffn.layer_norm."
    sd[last + "weight"] *= 2.0 ** -h
    sd[last + "bias"] *= 2.0 ** -h
    # PostNet: the BatchNorm's affine terms by 2^x scale the folded weight and bias by 2^x exactly (the tanh after takes it).  The folded
    # weight's header varies with the seed, so x takes it to post_ref[i] + h
    i = 0
    while f"postnet.convolutions.{i}.1.weight" in sd:
        h = nxt()
        x = (post_ref[i] if post_ref else _postnet_exponent(sd, i)) + h - _postnet_exponent(sd, i)
        sd[f"postnet.convolutions.{i}.1.weight"] *= 2.0 ** x
        sd[f"postnet.convolutions.{i}.1.bias"] *= 2.0 ** x
        i += 1
    # tables: position tables shifted by 3v (encoder) and 5v (decoder) positions, duration bias of 5 + v / 2 frames per phoneme,
    # bins stretched by 1 + v / 25
    for key, off in (("encoder.position_enc", 3 * v), ("decoder.position_enc", 5 * v)):
        _, rows, d = sd[key].shape
        sd[key] = synth.sinusoid_table(rows + off, d)[off:].unsqueeze(0).contiguous()
    sd["variance_adaptor.duration_predictor.linear_layer.bias"].fill_(math.log(5.0 + 0.5 * v + 1.0))
    for k in ("variance_adaptor.pitch_bins", "variance_adaptor.energy_bins"):
        sd[k] = sd[k] * (1.0 + v / 25)
    return sd


_CACHE = {}


def voice_state_dicts(pc, mc):
    """The 8 voices' state dicts (CPU), cached per config."""
    key = (pc["dataset"], mc["transformer"]["encoder_layer"], mc["transformer"]["decoder_layer"])
    if key not in _CACHE:
        base = synth.fastspeech2_state_dict(pc, mc, seed=SEEDS[0])
        n_post = sum(1 for k in base if k.startswith("postnet.convolutions.") and k.endswith(".1.weight"))
        ref = {i: _postnet_exponent(base, i) for i in range(n_post)}
        _CACHE[key] = [voice_state_dict(pc, mc, v, ref) for v in range(MAX_VOICES)]
    return _CACHE[key]


def packed_headers(sd, mc, tc_mask=None):
    """{packed tensor-core key: tuple of its weight-scale headers (1 / scale)} as FastSpeech2._pack packs sd under tc_mask (None: the
    default mask): one header per layer, one per segment of the K-segmented encoder and predictor convs."""
    tr = mc["transformer"]
    if tc_mask is None:
        tc_mask = L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8 | L.TC_ENCODER | L.TC_PREDICTORS
    n_post = sum(1 for k in sd if k.startswith("postnet.convolutions.") and k.endswith(".0.conv.weight"))
    pk = packing.pack_acoustic(lambda k: sd[k].float(), tr["encoder_layer"], tr["decoder_layer"], n_post, bool(mc["multi_speaker"]),
                               f8_decoder=bool(tc_mask & L.TC_DECODER_F8), f8_postnet=bool(tc_mask & L.TC_POSTNET_F8))
    out = {}
    for k, t in pk.items():
        if not k.endswith("_tc"):
            continue
        w = pk[k[:-3]]
        seg = k.startswith("enc.") or k.split(".")[0] in ("dur", "pitch", "energy")
        step = packing.TC_HEADER_BYTES + 1024 * w.shape[-1] if seg else t.numel()
        out[k] = tuple(float(t[o:o + 4].view(torch.float32)[0]) for o in range(0, t.numel(), step))
    return out


def check_state(sds):
    """AssertionError unless every state tensor a kernel reads differs between every pair of voices."""
    keys = [k for k in sds[0] if not k.endswith(UNREAD)]
    for a in range(len(sds)):
        for b in range(a + 1, len(sds)):
            same = [k for k in keys if torch.equal(sds[a][k], sds[b][k])]
            assert not same, f"voices {a} and {b} share {same[:4]}{'...' if len(same) > 4 else ''}"


def check_headers(sds, mc):
    """AssertionError unless every tensor-core layer's headers differ between every pair of voices, and every K-segmented conv has
    >= 2 distinct segment headers in each voice, in relative patterns that differ between voices as far as the segment count allows.
    Returns the voices' packed_headers."""
    hdrs = [packed_headers(sd, mc) for sd in sds]
    for k in hdrs[0]:
        per = [h[k] for h in hdrs]
        assert len(set(per)) == len(per), f"{k}: weight-scale headers shared between voices {per}"
        if len(per[0]) > 1:
            for v, h in enumerate(per):
                assert len(set(h)) >= 2, f"{k}: voice {v} has one header for all {len(h)} segments"
            rel = {tuple(round(math.log2(x / min(h))) for x in h) for h in per}
            want = min(len(per), (1 << len(per[0])) - 2)
            assert len(rel) >= want, f"{k}: {len(rel)} segment patterns over {len(per)} voices, want {want}"
    return hdrs


def check_voices(sds, mc):
    """check_state and check_headers."""
    check_state(sds)
    return check_headers(sds, mc)


def check_sane(sds, pc, mc, B=2, L_=24, seed=80):
    """Each voice through the CPU oracle on a small batch: finite mel, 3 to 15 frames per phoneme on average."""
    from oracle import fs2_oracle as O
    spk, texts, lens, Lm = synth.make_batch(B, L_, seed=seed, min_len=L_ // 2)
    for v, sd in enumerate(sds):
        out = O.fastspeech2_forward(sd, spk, texts, lens, Lm)
        assert torch.isfinite(out[0]).all() and torch.isfinite(out[1]).all(), v
        assert out[1].abs().max() < 1e3, (v, float(out[1].abs().max()))
        fpp = float(out[9].sum()) / float(lens.sum())
        assert 3.0 <= fpp <= 15.0, (v, fpp)


# ---------------------------------------------------------------- batches and plans

def postnet0_case(fmt, NG, T):
    """The PostNet's first conv (n_mel = 80 -> 512, k = 5, tanh) as a tests/conv_group_cases.py case: the one acoustic layer whose
    shape lets the planner group channel blocks (a single K-segment and Cin / 16 <= 8)."""
    return G.case(f"postnet0_{fmt}_ng{NG}", (), fmt, 80, 512, 5, NG, out_act=L.ACT_TANH, T=T)


# (mask name, operand format of the PostNet under it, NG, T): every NG the planner gives the PostNet's first conv in the two formats.
# T = 1000 is LJSpeech's max_seq_len: the decoder still reads each voice's own position table (a longer call recomputes the sinusoid
# table for every voice, so a solo call of a shorter utterance would read another table), and 1000 % 128 != 0 leaves a partial tile
GROUP_T = 1000
GROUP_TARGETS = [("default", "f8", 2, GROUP_T), ("default", "f8", 4, GROUP_T), ("default", "f8", 8, GROUP_T),
                 ("no_f8", "split3", 2, GROUP_T), ("no_f8", "split3", 4, GROUP_T)]


def forced_batch(B, L_, T, seed, min_len=None):
    """A batch with teacher-forced durations whose longest utterance has exactly T frames (utterance 0) and the others T / 2 to T:
    (speakers, texts, src_lens, max_src_len, mel_lens, d_targets)."""
    spk, texts, lens, Lm = synth.make_batch(B, L_, seed=seed, min_len=L_ // 2 if min_len is None else min_len)
    g = torch.Generator().manual_seed(seed)
    frames = torch.randint(T // 2, T + 1, (B,), generator=g)
    frames[0] = T
    d = torch.zeros(B, Lm, dtype=torch.long)
    for b in range(B):
        n, f = int(lens[b]), int(frames[b])
        d[b, :n] = f // n
        d[b, :f % n] += 1
    return spk, texts, lens, Lm, d.sum(1), d


def items(B, rows, T, groups):
    """The utterance of each work item of the tensor-core conv, in the kernel's order (channel-block group, utterance, tile):
    rows None for the padded batch (every utterance T rows), else the ragged batch's rows per utterance."""
    tiles = [-(-(T if rows is None else int(rows[b])) // 128) for b in range(B)]
    return [b for _ in range(groups) for b in range(B) for _ in range(tiles[b])]


def clashes(voice, seq, grid):
    """Consecutive work items of one persistent CTA (item i, i + grid) that belong to the same voice."""
    return sum(voice[seq[i]] == voice[seq[i + grid]] for i in range(len(seq) - grid))


def voice_mix(B, T, rows, plan):
    """A voice per utterance, all 8 present, such that no CTA runs two consecutive work items of one voice, padded or ragged; None if
    none of the mixes tried does."""
    groups = plan["n_items"] // plan["NG"] // (B * plan["tiles_per_batch"])
    seqs = [items(B, None, T, groups), items(B, rows, T, groups)]
    for m in (3, 5, 1, 7):
        for d in range(1, B + 1):
            voice = [(m * b + b // d) % MAX_VOICES for b in range(B)]
            if len(set(voice)) == MAX_VOICES and not any(clashes(voice, s, plan["grid"]) for s in seqs):
                return voice
    return None


GROUP_SEED = 90


def group_batch(fmt, NG, T, sms, seed=GROUP_SEED):
    """The PostNet's first conv in format fmt planned at NG on sms SMs: the smallest batch from conv_group_cases.choose_batch up at which
    the planner picks NG and a voice mix separates every CTA's consecutive items (a CTA steps `grid` items at a time, so at some B it
    meets the same utterance again), its teacher-forced inputs (48 phonemes per utterance) and the mix: (B, plan, forced_batch, voice)."""
    c = postnet0_case(fmt, NG, T)
    B0 = G.choose_batch(c, sms)
    for B in range(B0, B0 + 16):
        p = G.plan(c, B, sms)
        fb = forced_batch(B, 48, T, seed=seed + NG)
        voice = voice_mix(B, T, fb[4], p) if p["NG"] == NG else None
        if voice:
            return B, p, fb, voice
    raise AssertionError(f"{c['name']}: no batch from {B0} plans NG = {NG} with a voice mix on {sms} SMs")


# ---------------------------------------------------------------- the exact path's tiles

def simt_layers(B, L_, T, mc, n_mel=80):
    """The acoustic model's convs as the exact kernel runs them (tc_mask = 0): (name, B, rows, Cin, N, taps), the encoder and the
    phoneme-level predictors at L_ rows per utterance, the decoder, mel_linear and the PostNet at T."""
    tr, vp = mc["transformer"], mc["variance_predictor"]
    D, F, (k1, k2), VF = tr["encoder_hidden"], tr["conv_filter_size"], tr["conv_kernel_size"], vp["filter_size"]
    out = []
    for part, rows in (("encoder", L_), ("decoder", T)):
        out += [(f"{part}.qkv", B, rows, D, 3 * D, 1), (f"{part}.proj", B, rows, D, D, 1), (f"{part}.ffn.w_1", B, rows, D, F, k1),
                (f"{part}.ffn.w_2", B, rows, F, D, k2)]
    out += [("predictor.conv1", B, L_, D, VF, vp["kernel_size"]), ("predictor.conv2", B, L_, VF, VF, vp["kernel_size"]),
            ("mel_linear", B, T, D, n_mel, 1)]
    post = [(n_mel, 512)] + [(512, 512)] * 3 + [(512, n_mel)]
    out += [(f"postnet.{i}", B, T, ci, co, 5) for i, (ci, co) in enumerate(post)]
    return out


def simt_tile(B, rows, Cin, N, taps, sms):
    import ctypes
    a = L.Conv1dArgs(x=0x1000, x_batch_stride=rows * Cin, x_row_stride=Cin, B=B, T=rows, Cin=Cin, w=0x1000, N=N, taps=taps,
                     dilation=1, pad_left=(taps - 1) // 2, y=0x1000, y_batch_stride=rows * N, y_row_stride=N, alpha=1.0)
    out = L.ConvSimtPlan()
    assert L.lib().fs2_conv_simt_plan(ctypes.byref(a), sms, ctypes.byref(out)) == 0
    return (out.BM, out.BN)


def simt_tiles(shapes, mc, sms):
    """{(BM, BN)} fs2_conv_simt_plan gives the acoustic convs at the (B, L, T) shapes on sms SMs."""
    return {simt_tile(B, rows, ci, n, k, sms) for s in shapes for _, B, rows, ci, n, k in simt_layers(*s, mc)}


def simt_universe(mc, sms):
    """Every (BM, BN) fs2_conv_simt_plan gives an acoustic conv at any batch of 1 to 64 utterances of 1 to 2048 rows."""
    rows = sorted({1, 2048} | {1 << k for k in range(11)} | {(1 << k) + 1 for k in range(11)} | set(range(16, 400, 16)))
    return simt_tiles([(B, r, r) for B in (1, 2, 3, 4, 6, 8, 12, 16, 17, 24, 32, 48, 64) for r in rows], mc, sms)


# the exact path's batches: (B, phonemes, frames) with teacher-forced durations.  A single utterance gives the small grids' 64-row
# tiles and 64-column CTAs; 17 utterances add 64-row tiles at 128 columns (encoder and predictors) and 128-row tiles (decoder)
EXACT_SHAPES = [(1, 40, 300), (17, 48, 500)]
