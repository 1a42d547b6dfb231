"""CPU: the voices mode of the acoustic C ABI (fs2_acoustic_{encode,decode}_voices) and VoiceBank's host side, checked without a GPU:
struct layout, workspace bounds, every refusal made before any CUDA call, the bank's construction and argument checks, and the SASS of
the tensor-core conv's voices entry points."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.model import FastSpeech2, VoiceBank

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRY_POINTS = ("fs2_encode_voices_workspace_bytes", "fs2_decode_voices_workspace_bytes", "fs2_acoustic_encode_voices",
                "fs2_acoustic_decode_voices")


def test_struct_layout_matches_the_header(tmp_path):
    assert ctypes.sizeof(L.AcousticVoices) == L.ACOUSTIC_VOICES_SIZE == 32 and L.MAX_VOICES == 8
    offsets = {n: getattr(L.AcousticVoices, n).offset for n, _ in L.AcousticVoices._fields_}
    assert offsets == {"n": 0, "models": 8, "models_dev": 16, "voice": 24}
    h = L.lib()
    for name in ENTRY_POINTS:
        assert name in L.EXPORTS and getattr(h, name).argtypes == L.EXPORTS[name][1]
    assert h.fs2_abi_version() == L.ABI_VERSION == 12
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to read the header's layout")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fs2b200.h"\nint main(void) { printf("%zu %zu %zu %zu %zu %d\\n", '
                   "sizeof(fs2_acoustic_voices), offsetof(fs2_acoustic_voices, n), offsetof(fs2_acoustic_voices, models), "
                   "offsetof(fs2_acoustic_voices, models_dev), offsetof(fs2_acoustic_voices, voice), FS2_MAX_VOICES); return 0; }\n")
    exe = tmp_path / "layout"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [32, offsets["n"], offsets["models"], offsets["models_dev"], offsets["voice"], L.MAX_VOICES]


def _model(**kw):
    """An LJSpeech-shaped struct whose every weight pointer is a fake, 16-byte aligned address (no CUDA call reads it)"""
    m = L.AcousticModel(d_model=256, n_head=2, d_inner=1024, k1=9, k2=1, n_enc=4, n_dec=6, n_mel=80, vp_filter=256, vp_kernel=3,
                        n_bins=256, n_vocab=361, enc_pos_rows=1001, dec_pos_rows=1001, n_postnet=5, post_k=5,
                        tc_mask=L.TC_DECODER | L.TC_POSTNET | L.TC_ENCODER | L.TC_PREDICTORS)
    addr = iter(range(0x10000, 0x10000 + 16 * 4096, 16))
    for name in ("word_emb", "enc_pos", "dec_pos", "pitch_bins", "energy_bins", "pitch_emb", "energy_emb", "w_mel", "b_mel", "w_mel_tc"):
        setattr(m, name, next(addr))
    for side in (m.enc[:4], m.dec[:6]):
        for blk in side:
            for name, _ in L.FftBlockWeights._fields_:
                setattr(blk, name, next(addr))
    for pred in (m.dur, m.pitch, m.energy):
        for name, _ in L.PredictorWeights._fields_:
            setattr(pred, name, next(addr))
    for i in range(5):
        m.post_cin[i], m.post_cout[i] = (80 if i == 0 else 512), (80 if i == 4 else 512)
        m.w_post[i], m.b_post[i], m.w_post_tc[i] = next(addr), next(addr), next(addr)
    for k, v in kw.items():
        setattr(m, k, v)
    return m


def _voices(models, n=None, models_dev=0x2000, voice=0x3000):
    arr = L.acoustic_model_array(models)
    v = L.AcousticVoices(n=len(models) if n is None else n, models=ctypes.addressof(arr), models_dev=models_dev, voice=voice)
    v._arr = arr
    return v


def _encode_args(**kw):
    base = dict(B=3, L=40, texts=0x1000, src_lens=0x1000, logd_pred=0x1000, d_rounded=0x1000, mel_lens=0x1000, cum_dur=0x1000,
                x_adapted=0x1000, len_stats=0x1000, workspace=0x1000, workspace_bytes=1)
    base.update(kw)
    return L.EncodeArgs(**base)


def _decode_args(**kw):
    base = dict(B=3, L=40, T=300, x_adapted=0x1000, cum_dur=0x1000, mel_mask_lens=0x1000, mel=0x1000, postnet_mel=0x1000,
                workspace=0x1000, workspace_bytes=1)
    base.update(kw)
    return L.DecodeArgs(**base)


def test_workspace_is_the_single_model_bound_plus_the_staged_table():
    h = L.lib()
    models = [_model(), _model()]
    v = _voices(models)
    for B, n in ((1, 7), (3, 40), (64, 256), (65, 1000)):
        table = (2 * B * 4 + 255) // 256 * 256            # [2B] int32, one 256-byte-aligned allocation
        assert h.fs2_encode_voices_workspace_bytes(ctypes.byref(v), B, n) == h.fs2_encode_workspace_bytes(ctypes.byref(models[0]), B, n) + table
        assert h.fs2_decode_voices_workspace_bytes(ctypes.byref(v), B, n) == h.fs2_decode_workspace_bytes(ctypes.byref(models[0]), B, n) + table
    assert h.fs2_encode_voices_workspace_bytes(ctypes.byref(_voices(models, n=0)), 3, 40) == 0
    assert h.fs2_decode_voices_workspace_bytes(ctypes.byref(_voices([models[0], _model(n_bins=128)])), 3, 40) == 0


def _layout_breakers():
    """(name, voice 1's struct) pairs that differ from _model() in one int field, a tile's presence, or an address mod 16"""
    out = [(f, _model(**{f: getattr(_model(), f) + 1})) for f in
           ("d_model", "d_inner", "k1", "k2", "n_enc", "n_dec", "n_mel", "vp_filter", "vp_kernel", "n_bins", "n_vocab", "n_speakers",
            "pitch_frame_level", "energy_frame_level", "n_postnet", "post_k")]
    out.append(("n_head", _model(n_head=4)))
    out.append(("tc_mask", _model(tc_mask=0)))
    m = _model()
    m.post_cout[1] = 256
    out.append(("post_cout", m))
    m = _model()
    m.enc[2].w_1_tc = 0
    out.append(("tile NULL", m))
    ref = _model()
    ref.w_mel_tc = 0
    out.append(("tile non-NULL", (ref, _model())))        # voice 0 without the tile, voice 1 with it
    m = _model()
    m.pitch.w_out += 8
    out.append(("address + 8", m))
    m = _model()
    m.w_post_tc[3] += 8
    out.append(("tile address + 8", m))
    return out


def test_every_refusal_comes_before_any_cuda_call():
    """Every pointer is fake: FS2_ERR_ARG must come from host checks (a CUDA call would fail differently or crash)."""
    h = L.lib()
    ref = ctypes.byref
    m0 = _model()
    good = [m0, _model()]
    cases = [_voices(good, n=0), _voices(good * 5, n=9), _voices(good, models_dev=0), _voices(good, voice=0),
             _voices([m0, _model(enc_pos_rows=39)]), _voices([m0, _model(dec_pos_rows=299)])]
    nulls = L.AcousticVoices(n=2, models=0, models_dev=0x2000, voice=0x3000)
    cases.append(nulls)
    for name, m in _layout_breakers():
        pair = list(m) if isinstance(m, tuple) else [m0, m]
        cases.append(_voices(pair))
    for i, v in enumerate(cases):
        # case 4 has short encoder positions only, case 5 short decoder positions only: each is called on that phase alone
        if i != 5:
            assert h.fs2_acoustic_encode_voices(ref(v), ref(_encode_args()), None, 0, None) == -1, i
        if i != 4:
            assert h.fs2_acoustic_decode_voices(ref(v), ref(_decode_args()), None, 1, None) == -1, i
    v = _voices(good)
    for ragged in (-1, 2):
        assert h.fs2_acoustic_encode_voices(ref(v), ref(_encode_args()), None, ragged, None) == -1
        assert h.fs2_acoustic_decode_voices(ref(v), ref(_decode_args()), None, ragged, None) == -1
    assert h.fs2_acoustic_encode_voices(None, ref(_encode_args()), None, 0, None) == -1
    assert h.fs2_acoustic_encode_voices(ref(v), None, None, 0, None) == -1
    # a short workspace is refused before any launch, as in the single-model call
    need = h.fs2_encode_voices_workspace_bytes(ref(v), 3, 40)
    assert h.fs2_acoustic_encode_voices(ref(v), ref(_encode_args(workspace_bytes=need - 257)), None, 0, None) == -3


# --------------------------------------------------------------------------------------------------------------- VoiceBank (host side)
@pytest.fixture(scope="module")
def lj(tmp_path_factory):
    return configs.make_configs("LJSpeech", str(tmp_path_factory.mktemp("vb")))


def _fs2(cfgs, seed=0):
    m = FastSpeech2(*cfgs)
    m.load_state_dict(synth.fastspeech2_state_dict(*cfgs, seed=seed))
    return m.eval()


def test_bank_construction_refusals(lj, libri_configs):
    a, b = _fs2(lj, 1), _fs2(lj, 2)
    VoiceBank([a, b])
    with pytest.raises(ValueError):
        VoiceBank([])
    with pytest.raises(ValueError):
        VoiceBank([a] * (L.MAX_VOICES + 1))
    with pytest.raises(ValueError):
        VoiceBank([a, _fs2(libri_configs)])                # another config
    c = _fs2(lj, 3)
    c.tc_mask = 0
    with pytest.raises(ValueError):
        VoiceBank([a, c])
    with pytest.raises(ValueError):
        VoiceBank([a, _fs2(lj, 4).train()])
    with pytest.raises(ValueError):
        VoiceBank([a, object()])


def test_bank_voice_argument_refusals(lj):
    bank = VoiceBank([_fs2(lj, 1), _fs2(lj, 2)])
    spk, texts, lens, Lm = synth.make_batch(3, 12, seed=0, min_len=4)
    for voice in (torch.tensor([0, 1]), torch.tensor([[0, 1, 0]]), torch.tensor([0., 1., 0.]), torch.tensor([True, False, True]),
                  [0, 1, 0], torch.tensor([0, 2, 1]), torch.tensor([-1, 0, 1])):
        with pytest.raises(ValueError):
            bank(voice, spk, texts, lens, Lm)


def test_bank_in_training_mode_raises(lj):
    a, b = _fs2(lj, 1), _fs2(lj, 2)
    bank = VoiceBank([a, b])
    b.train()
    spk, texts, lens, Lm = synth.make_batch(2, 12, seed=0, min_len=4)
    with pytest.raises(NotImplementedError):
        bank(torch.tensor([0, 1]), spk, texts, lens, Lm)


# --------------------------------------------------------------------------------------------------------------- SASS of the entry points
def test_offline_table_conv_entry_points_are_pipelined_and_do_not_spill():
    from tests.test_sass_pipeline import mmas_and_full_waits, res_usage_of, sass_of
    keep = re.compile(r"\dconv_tc_table_kernelILi\d+ELb[01]ELb0E").search     # the offline ones: conv_tc_table_kernel<NB, RAG, false>
    sass, usage = sass_of(keep), res_usage_of(keep)
    assert len(sass) == 16 and set(usage) == set(sass)       # 8 NB x (padded, ragged)
    for f, text in sass.items():
        mmas, full_waits = mmas_and_full_waits(text)
        assert mmas > 0 and full_waits * 4 <= mmas, (f, mmas, full_waits)
        assert usage[f]["STACK"] == 0 and usage[f]["LOCAL"] == 0, (f, usage[f])
