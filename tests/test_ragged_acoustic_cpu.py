"""CPU: the ragged acoustic entry points of the C ABI (fs2_acoustic_encode_ragged / fs2_acoustic_decode_ragged) and the drop-in's
--ragged flag, checked without a GPU."""
import ctypes
import os
import subprocess
import sys

from fastspeech2_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

STRUCTS = (_lib.Conv1dArgs, _lib.LayerNormArgs, _lib.AttentionArgs, _lib.EmbedArgs, _lib.RowBiasArgs, _lib.VarianceHeadArgs,
           _lib.DurationsArgs, _lib.LengthRegulateArgs, _lib.ConvPostArgs, _lib.AcousticModel, _lib.EncodeArgs, _lib.DecodeArgs,
           _lib.VocoderModel, _lib.VocoderArgs, _lib.ResstackArgs, _lib.WavInt16Args, _lib.ConvTcPlan, _lib.ConvSimtPlan, _lib.ResstackPlan)


def test_ragged_entry_points_are_bound_and_the_abi_is_unchanged():
    h = _lib.lib()
    for name in ("fs2_acoustic_encode_ragged", "fs2_acoustic_decode_ragged"):
        assert name in _lib.EXPORTS and getattr(h, name).argtypes == _lib.EXPORTS[name][1]
    assert h.fs2_abi_version() == _lib.ABI_VERSION == 12
    for i, cls in enumerate(STRUCTS):
        assert h.fs2_struct_size(i) == ctypes.sizeof(cls), cls.__name__
    assert h.fs2_struct_size(len(STRUCTS)) == 0


def _model(d_model=256, n_head=2):
    m = _lib.AcousticModel(d_model=d_model, n_head=n_head, d_inner=1024, k1=9, k2=1, n_enc=4, n_dec=6, n_mel=80, vp_filter=256,
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


def test_invalid_arguments_are_refused_before_any_cuda_call():
    """Every pointer below is fake: the refusals come from host checks, and each returns the default entry point's error code."""
    h = _lib.lib()
    m = _model()
    ref = ctypes.byref
    for ragged, default in ((h.fs2_acoustic_encode_ragged, h.fs2_acoustic_encode), (h.fs2_acoustic_decode_ragged, h.fs2_acoustic_decode)):
        make = _encode_args if ragged is h.fs2_acoustic_encode_ragged else _decode_args
        cases = [(None, make()), (m, None), (m, make(B=0)), (m, make(L=0)),
                 (m, make(workspace=0)), (_model(n_head=4), make()), (_model(d_model=0), make())]
        if make is _encode_args:
            cases += [(m, make(texts=0)), (m, make(src_lens=0)), (m, make(d_rounded=0))]
        else:
            cases += [(m, make(T=0)), (m, make(mel_mask_lens=0)), (m, make(postnet_mel=0))]
        for model, args in cases:
            rc = ragged(ref(model) if model is not None else None, ref(args) if args is not None else None, None)
            assert rc in (-1, -2) and rc == default(ref(model) if model is not None else None, ref(args) if args is not None else None, None)


def test_ragged_calls_take_the_default_workspace_sizes():
    """There is one workspace query per phase: a ragged call refuses exactly the sizes the default call refuses (FS2_ERR_WORKSPACE is
    decided before any launch)."""
    h = _lib.lib()
    m = _model()
    need_e = h.fs2_encode_workspace_bytes(ctypes.byref(m), 3, 40)
    need_d = h.fs2_decode_workspace_bytes(ctypes.byref(m), 3, 300)
    assert need_e > 0 and need_d > 0
    for have in (1, need_e // 2, need_e - 257):
        a = _encode_args(workspace_bytes=have)
        assert h.fs2_acoustic_encode_ragged(ctypes.byref(m), ctypes.byref(a), None) == -3
        assert h.fs2_acoustic_encode(ctypes.byref(m), ctypes.byref(a), None) == -3
    for have in (1, need_d // 2, need_d - 257):
        a = _decode_args(workspace_bytes=have)
        assert h.fs2_acoustic_decode_ragged(ctypes.byref(m), ctypes.byref(a), None) == -3
        assert h.fs2_acoustic_decode(ctypes.byref(m), ctypes.byref(a), None) == -3


_FAKE_REFERENCE = r'''
import sys, functools
import utils.model as um
import model
print("ARGV", sys.argv[1:])
v = um.vocoder_infer
ragged = isinstance(v, functools.partial) and v.keywords == {"ragged": True}
print("RAGGED", ragged, "ACOUSTIC", model.FastSpeech2.ragged)
'''


def _run_main(tmp_path, args, script_text):
    (tmp_path / "utils").mkdir(exist_ok=True)
    (tmp_path / "utils" / "__init__.py").write_text("")
    (tmp_path / "utils" / "model.py").write_text("def vocoder_infer(*a, **k):\n    raise AssertionError('not patched')\n")
    script = tmp_path / "synthesize.py"
    script.write_text(script_text)
    code = "import sys; sys.path.insert(0, %r)\nimport fastspeech2_b200.dropin as d\nd.main(%r)\n" % (ROOT, [a if a != "SCRIPT" else str(script) for a in args])
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def test_dropin_main_ragged_flag_sets_both_modes(tmp_path):
    import fastspeech2_b200.model as b_model
    assert b_model.FastSpeech2.ragged is False
    out = _run_main(tmp_path, ["--ragged", "SCRIPT", "--mode", "batch", "--ragged"], _FAKE_REFERENCE)
    assert "ARGV ['--mode', 'batch', '--ragged']" in out       # flags after the script path belong to the script
    assert "RAGGED True ACOUSTIC True" in out
    out = _run_main(tmp_path, ["--ragged-vocoder", "SCRIPT", "--ragged"], _FAKE_REFERENCE)
    assert "ARGV ['--ragged']" in out and "RAGGED True ACOUSTIC False" in out
    out = _run_main(tmp_path, ["SCRIPT", "--mode", "single"], _FAKE_REFERENCE)
    assert "ARGV ['--mode', 'single']" in out and "RAGGED False ACOUSTIC False" in out
