"""CPU: tensor-valued p_control / d_control (per utterance [B, 1], per phoneme [B, L]).  The oracle against the reference's own outputs
(tests/golden/fs2_controls.npz, oracle/gen_golden_controls.py), the host-side normaliser of FastSpeech2.forward, and the C ABI's
fs2_acoustic_{encode,decode}_ctl argument checks -- none of it needs a GPU."""
import ctypes
import os

import numpy as np
import pytest
import torch

from fastspeech2_b200 import _lib, configs, synth
from fastspeech2_b200.model.fastspeech2 import normalize_control
from oracle import fs2_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
CASES = ("lj_utt", "lj_phoneme", "libri_utt", "paper_utt_phoneme")


def load_case(name, scratch):
    """(state_dict, inputs, controls, reference 10-tuple as tensors, frame_level) of one case of fs2_controls.npz"""
    from oracle.gen_golden import paper_state_dict
    z = np.load(os.path.join(GOLD, "fs2_controls.npz"))
    g = lambda k: z[f"{name}__{k}"]
    ds = str(g("dataset"))
    pc, mc = configs.make_configs(ds, scratch)
    sd = paper_state_dict(pc, mc, int(g("seed"))) if ds == "LJSpeech_paper" else synth.fastspeech2_state_dict(pc, mc, seed=int(g("seed")))
    t = lambda k: torch.from_numpy(g(k))
    inputs = (t("speakers"), t("texts"), t("src_lens"), int(g("max_src_len")))
    ctl = dict(p_control=t("p_control"), d_control=t("d_control"), e_control=t("e_control"))
    want = [t(k) for k in ("mel", "postnet_mel", "p_pred", "e_pred", "logd", "d_rounded", "src_masks", "mel_masks", "src_lens_out",
                           "mel_lens")]
    return (pc, mc), sd, inputs, ctl, want, ds == "LJSpeech_paper"


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference_with_tensor_controls(name, scratch):
    _, sd, inputs, ctl, want, frame = load_case(name, scratch)
    assert ctl["p_control"].numel() > 1 and ctl["d_control"].numel() > 1
    lv = dict(pitch_level="frame_level", energy_level="frame_level") if frame else {}
    out = O.fastspeech2_forward(sd, *inputs, **ctl, **lv)
    assert torch.equal(out[5], want[5]) and torch.equal(out[9], want[9])
    assert torch.equal(out[6], want[6]) and torch.equal(out[7], want[7])
    for i in (0, 1, 4):
        assert (out[i] - want[i]).abs().max() < 5e-6, i
    for i in (2, 3):           # the paper config's raw-valued heads: relative, as test_oracle_golden
        assert ((out[i] - want[i]).abs() / ((1 + want[i].abs()) if frame else 1)).max() < 5e-6 * (10 if frame else 1), i
    # the controls did something: the same inputs with unit controls give other durations
    plain = O.fastspeech2_forward(sd, *inputs, **lv)
    assert not torch.equal(plain[5], want[5])


# ------------------------------------------------------------------------------------------------------------ normaliser
B, L, T = 3, 5, 11


@pytest.mark.parametrize("make", [
    lambda: torch.rand(B, 1), lambda: torch.rand(B, L), lambda: torch.rand(1, L), lambda: torch.rand(L), lambda: torch.tensor(1.5),
    lambda: torch.rand(B, 1).expand(B, L), lambda: torch.rand(L).expand(B, L), lambda: torch.rand(L, B).t(),
    lambda: torch.rand(B, L, dtype=torch.float64), lambda: torch.randint(1, 3, (B, 1)), lambda: torch.rand(B, L, dtype=torch.float16),
    lambda: 1.25, lambda: 2, lambda: torch.rand(1, 1, 1)])
def test_normaliser_accepts_what_broadcasts_to_the_prediction(make):
    c = make()
    t, scalar, strides = normalize_control(c, (B, L), torch.device("cpu"))
    if not torch.is_tensor(c) or c.numel() == 1:                       # today's scalar path
        assert t is None and scalar == float(c)
        return
    want = c.to(torch.float32).broadcast_to((B, L))
    assert scalar == 1.0 and t.dtype == torch.float32 and tuple(t.shape) == (B, L) and strides == t.stride()
    assert torch.equal(t, want)
    flat = t.as_strided((t.untyped_storage().nbytes() // 4,), (1,), 0)   # what the kernel sees: v[b * sb + l * sl]
    for b in range(B):
        for l in range(L):
            assert flat[t.storage_offset() + b * strides[0] + l * strides[1]] == want[b, l]
    for s, n in zip(strides, torch.broadcast_shapes(c.shape, (1, 1))):
        assert n > 1 or s == 0                                         # broadcast dimensions are not materialised


def test_normaliser_does_not_materialise_an_expanded_view():
    c = torch.rand(B, 1, dtype=torch.float64).expand(B, L)
    t, _, strides = normalize_control(c, (B, L), torch.device("cpu"))
    assert strides == (1, 0) and t.untyped_storage().nbytes() == B * 4


@pytest.mark.parametrize("shape,pred,why", [
    ((B,), (B, L), "does not broadcast"),                 # 1-D is per column (the phoneme axis), as in the reference
    ((L, L, 1), (L, L), "would grow"),                    # [B, L, 1] with B == L: the reference would silently grow every later tensor
    ((B, L, 1), (B, L), "does not broadcast"),
    ((B, 1, 1), (B, L), "would grow"),
    ((B, L), (B, T), "does not broadcast"),               # per-phoneme p_control of a frame-level predictor
    ((2, L), (B, L), "does not broadcast"),
    ((1, B, L), (B, L), "would grow")])
def test_normaliser_rejects_what_the_reference_rejects_or_grows(shape, pred, why):
    with pytest.raises(ValueError, match=why):
        normalize_control(torch.rand(*shape), pred, torch.device("cpu"), "p_control")
    if why == "does not broadcast":                       # the reference's `prediction * control` raises too
        with pytest.raises(RuntimeError):
            torch.rand(*pred) * torch.rand(*shape)
    else:                                                 # the reference's product has another shape than the prediction
        assert (torch.rand(*pred) * torch.rand(*shape)).shape != pred


def test_normaliser_per_utterance_b_equals_l_is_still_per_column():
    c = torch.arange(1.0, 4.0)                            # [B] with B == L: the reference scales phonemes, so does this
    t, _, _ = normalize_control(c, (3, 3), torch.device("cpu"))
    assert torch.equal(t, c.expand(3, 3)) and not torch.equal(t, c[:, None].expand(3, 3))


def test_normaliser_rejects_complex():
    with pytest.raises(ValueError, match="real"):
        normalize_control(torch.ones(B, L, dtype=torch.complex64), (B, L), torch.device("cpu"))


# ------------------------------------------------------------------------------------------------------------ C ABI
def test_control_struct_layout_and_binding():
    h = _lib.lib()
    assert ctypes.sizeof(_lib.ControlArgs) == 48                     # static_assert(sizeof(fs2_control_args) == 48) in model.cu
    assert [f[0] for f in _lib.ControlArgs._fields_] == ["p", "p_stride_b", "p_stride_l", "d", "d_stride_b", "d_stride_l"]
    for name in ("fs2_acoustic_encode_ctl", "fs2_acoustic_decode_ctl"):
        assert getattr(h, name).argtypes == _lib.EXPORTS[name][1]
    assert h.fs2_abi_version() == 12


def _model(n_head=2):
    m = _lib.AcousticModel(d_model=256, n_head=n_head, d_inner=1024, k1=9, k2=1, n_enc=4, n_dec=6, n_mel=80, vp_filter=256,
                           vp_kernel=3, n_bins=256, n_vocab=361, enc_pos_rows=1001, dec_pos_rows=1001, n_postnet=5, post_k=5)
    for i in range(5):
        m.post_cin[i], m.post_cout[i] = (80 if i == 0 else 512), (80 if i == 4 else 512)
    return m


def _encode_args(**kw):
    base = dict(B=3, L=40, texts=0x1000, src_lens=0x1000, logd_pred=0x1000, d_rounded=0x1000, mel_lens=0x1000, cum_dur=0x1000,
                x_adapted=0x1000, len_stats=0x1000, workspace=0x1000, workspace_bytes=1)
    base.update(kw)
    return _lib.EncodeArgs(**base)


def _decode_args(**kw):
    base = dict(B=3, L=40, T=300, x_adapted=0x1000, cum_dur=0x1000, mel_mask_lens=0x1000, mel=0x1000, postnet_mel=0x1000,
                workspace=0x1000, workspace_bytes=1)
    base.update(kw)
    return _lib.DecodeArgs(**base)


def test_ctl_host_side_argument_checks_need_no_gpu():
    """Every pointer is fake: the refusals come from host checks before any CUDA call.  Without controls (ctl NULL or both pointers
    NULL) a _ctl call returns what the entry point without controls returns; bad controls or a ragged flag other than 0 / 1 are
    FS2_ERR_ARG."""
    h = _lib.lib()
    ref = ctypes.byref
    m = _model()
    null_ctl = _lib.ControlArgs()
    good = _lib.ControlArgs(p=0x1000, p_stride_b=40, p_stride_l=1, d=0x1000, d_stride_b=0, d_stride_l=1)
    phases = ((h.fs2_acoustic_encode_ctl, h.fs2_acoustic_encode, h.fs2_acoustic_encode_ragged, _encode_args),
              (h.fs2_acoustic_decode_ctl, h.fs2_acoustic_decode, h.fs2_acoustic_decode_ragged, _decode_args))
    for ctl_fn, default, ragged_fn, make in phases:
        cases = [(None, make()), (m, None), (m, make(B=0)), (m, make(L=0)), (m, make(workspace=0)), (_model(n_head=4), make()),
                 (m, make())]                          # the last: a workspace of one byte, FS2_ERR_WORKSPACE
        for model, args in cases:
            mp, ap = (ref(model) if model is not None else None), (ref(args) if args is not None else None)
            for rg, plain in ((0, default), (1, ragged_fn)):
                want = plain(mp, ap, None)
                assert want in (-1, -2, -3)
                assert ctl_fn(mp, ap, None, rg, None) == want
                assert ctl_fn(mp, ap, ref(null_ctl), rg, None) == want
                assert ctl_fn(mp, ap, ref(good), rg, None) == want
        for bad in (dict(p_stride_b=-1), dict(p_stride_l=-40), dict(d_stride_b=-1), dict(d_stride_l=-1)):
            c = _lib.ControlArgs(p=0x1000, d=0x1000, **bad)
            assert ctl_fn(ref(m), ref(make()), ref(c), 0, None) == -1
        for rg in (-1, 2):
            assert ctl_fn(ref(m), ref(make()), None, rg, None) == -1
