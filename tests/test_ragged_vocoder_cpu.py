"""CPU: the ragged-vocoder additions to the C ABI (per-utterance lengths on fs2_conv1d / fs2_resstack / fs2_conv_post /
fs2_vocoder_forward) and the drop-in's --ragged-vocoder flag, checked without a GPU."""
import ctypes
import os
import subprocess
import sys

from fastspeech2_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ragged_fields_are_appended_and_sizes_match():
    h = _lib.lib()
    assert h.fs2_abi_version() == _lib.ABI_VERSION == 11
    for i, cls, tail in ((0, _lib.Conv1dArgs, ["x_lens", "lens_scale"]), (8, _lib.ConvPostArgs, ["lens", "lens_scale"]),
                         (13, _lib.VocoderArgs, ["mel_lens"]), (14, _lib.ResstackArgs, ["lens", "lens_scale"])):
        names = [f[0] for f in cls._fields_]
        assert names[-len(tail):] == tail, cls.__name__          # appended: positional construction of the old fields still works
        assert h.fs2_struct_size(i) == ctypes.sizeof(cls), cls.__name__


def test_lens_scale_below_one_is_refused_before_any_cuda_call():
    h = _lib.lib()
    lens = 0x2000                                               # never dereferenced: the check comes first
    for backend in (_lib.CONV_AUTO, _lib.CONV_SIMT, _lib.CONV_TC):
        for scale in (0, -1):
            a = _lib.Conv1dArgs(x=0x1000, x_batch_stride=64 * 32, x_row_stride=32, B=2, T=64, Cin=32, w=0x1000, N=32, taps=3,
                                pad_left=1, w_tc=0x1000, backend=backend, alpha=1.0, y=0x1000, y_batch_stride=64 * 32, y_row_stride=32,
                                x_lens=lens, lens_scale=scale)
            assert h.fs2_conv1d(ctypes.byref(a), None) == -1, (backend, scale)
    r = _lib.ResstackArgs(x=0x10000, y=0x40000, B=2, N=100, C=32, n_kernels=1, n_dil=1, lens=lens, lens_scale=0)
    r.k[0] = 3
    r.dil[0][0] = 1
    assert h.fs2_resstack(ctypes.byref(r), None) == -1
    p = _lib.ConvPostArgs(x=0x1000, B=2, T=64, C=32, w=0x1000, bias=0x1000, taps=7, in_slope=0.01, wav=0x1000, lens=lens, lens_scale=0)
    assert h.fs2_conv_post(ctypes.byref(p), None) == -1


def test_launch_plans_do_not_depend_on_lengths():
    """The host never reads device lengths: both plans size the grid from the padded shape, with or without lengths."""
    h = _lib.lib()
    for lens, scale in ((0, 0), (0x2000, 1), (0x2000, 256)):
        a = _lib.Conv1dArgs(x=0x1000, x_batch_stride=4096 * 64, x_row_stride=64, B=3, T=4096, Cin=64, w=0x1000, N=64, taps=7,
                            pad_left=3, w_tc=0x1000, alpha=1.0, y=0x1000, y_batch_stride=4096 * 64, y_row_stride=64,
                            tc_variant=_lib.TC_VARIANT_F8, x_lens=lens, lens_scale=scale)
        out = (ctypes.c_int32 * 11)()
        assert h.fs2_conv_tc_plan(ctypes.byref(a), 132, out) == 0
        r = _lib.ResstackArgs(x=0x10000, y=0x40000, B=3, N=4096, C=64, n_kernels=3, n_dil=3, lens=lens, lens_scale=scale)
        for j, k in enumerate((3, 7, 11)):
            r.k[j] = k
            for d, dv in enumerate((1, 3, 5)):
                r.dil[j][d] = dv
        rp = (ctypes.c_int32 * 12)()
        assert h.fs2_resstack_plan(ctypes.byref(r), 132, rp) == 0
        if lens == 0:
            ref_conv, ref_rs = list(out), list(rp)
        assert list(out) == ref_conv and list(rp) == ref_rs
    assert ref_conv[8] == 3 * 32 and ref_conv[9] == 96         # 3 x 32 tiles of one 64-channel block: padded shape
    assert ref_rs[3] == 3 * -(-4096 // ref_rs[2])


_FAKE_REFERENCE = r'''
import sys, functools
import utils.model as um
print("ARGV", sys.argv[1:])
v = um.vocoder_infer
ragged = isinstance(v, functools.partial) and v.keywords == {"ragged": True}
print("RAGGED", ragged, (v.func if ragged else v).__module__)
'''


def _run_main(tmp_path, args):
    (tmp_path / "utils").mkdir(exist_ok=True)
    (tmp_path / "utils" / "__init__.py").write_text("")
    (tmp_path / "utils" / "model.py").write_text("def vocoder_infer(*a, **k):\n    raise AssertionError('not patched')\n")
    script = tmp_path / "synthesize.py"
    script.write_text(_FAKE_REFERENCE)
    code = "import sys; sys.path.insert(0, %r)\nimport fastspeech2_b200.dropin as d\nd.main(%r)\n" % (ROOT, [a if a != "SCRIPT" else str(script) for a in args])
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def test_dropin_main_consumes_the_ragged_vocoder_flag(tmp_path):
    out = _run_main(tmp_path, ["--ragged-vocoder", "SCRIPT", "--mode", "batch", "--ragged-vocoder"])
    assert "ARGV ['--mode', 'batch', '--ragged-vocoder']" in out     # flags after the script path belong to the script
    assert "RAGGED True fastspeech2_b200.dropin" in out
    out = _run_main(tmp_path, ["SCRIPT", "--mode", "single"])
    assert "ARGV ['--mode', 'single']" in out and "RAGGED False fastspeech2_b200.dropin" in out
