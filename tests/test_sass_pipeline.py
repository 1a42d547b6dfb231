"""The wgmma pipelines of the tensor-core kernels, checked in the SASS of the built library (no GPU needed).

conv_tc_kernel, resstack_kernel and attention_fused_kernel keep several wgmma groups in flight: a weight stage is released one
commit group late (wgmma.wait_group 1), so the tensor core has the next stage's MMAs queued while the previous ones retire.  That
only holds if ptxas sees the MMAs in warp-uniform control flow.  When it does not (warning C7520), it wraps every MMA in its own
warpgroup arrive + full wait (`WARPGROUP.DEPBAR.LE gsb0, 0x0`): the code still computes the same thing, several times slower, and
the extra live ranges push the 96-register conv kernels into local-memory spills.  Nothing but the SASS shows it, so it is checked
here: per kernel, full waits must be rare next to the MMAs, and the conv kernels must not spill.  The parser below also serves the
SASS checks of the table mode's entry points (test_stream_multi_cpu.py, test_acoustic_voices_cpu.py).
"""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "fastspeech2_b200", "libfs2b200.so")
KERNELS = ("conv_tc_kernel", "resstack_kernel", "attention_fused_kernel")
N_INSTANTIATIONS = {"conv_tc_kernel": 16, "resstack_kernel": 4, "attention_fused_kernel": 2}


def _cuobjdump():
    found = shutil.which("cuobjdump")
    if found:
        return found
    for home in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if home and os.path.isfile(os.path.join(home, "bin", "cuobjdump")):
            return os.path.join(home, "bin", "cuobjdump")
    return None


def _dump(flag):
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    if not os.path.isfile(LIB):
        pytest.skip("libfs2b200.so has not been built")
    return subprocess.run([tool, flag, LIB], capture_output=True, text=True, check=True).stdout


def sass_of(keep):
    """{mangled name: SASS text} of every function of the library whose mangled name keep(name) accepts"""
    funcs, name = {}, None
    for line in _dump("-sass").splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if keep(m.group(1)) else None
            if name:
                funcs[name] = []
        elif name:
            funcs[name].append(line)
    return {k: "\n".join(v) for k, v in funcs.items()}


def res_usage_of(keep):
    """{mangled name: {resource: value}} of every function of the library whose mangled name keep(name) accepts"""
    out, name = {}, None
    for line in _dump("-res-usage").splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1) if keep(m.group(1)) else None
        elif name and "REG:" in line:
            out[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            name = None
    return out


def mmas_and_full_waits(text):
    """wgmma instructions and full wgmma waits in one function's SASS; pipelined: one full wait per accumulator hand-off to an
    epilogue, a handful per kernel (full_waits * 4 <= mmas); serialised: one per MMA"""
    return len(re.findall(r"\b[HQ]GMMA\.", text)), len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", text))


def _kernel(mangled):
    return next((k for k in KERNELS if k in mangled), None)


@pytest.fixture(scope="module")
def sass():
    """{mangled name: SASS text} of every tensor-core kernel"""
    return sass_of(_kernel)


@pytest.fixture(scope="module")
def res_usage():
    """{mangled name: {resource: value}} of every tensor-core kernel"""
    return res_usage_of(_kernel)


def test_every_instantiation_is_found(sass, res_usage):
    for kernel, n in N_INSTANTIATIONS.items():
        assert sum(_kernel(f) == kernel for f in sass) == n, kernel
        assert sum(_kernel(f) == kernel for f in res_usage) == n, kernel


@pytest.mark.parametrize("kernel", KERNELS)
def test_mmas_are_not_serialised(sass, kernel):
    for name, text in sass.items():
        if _kernel(name) != kernel:
            continue
        mmas, full_waits = mmas_and_full_waits(text)
        assert mmas > 0, name
        assert full_waits * 4 <= mmas, f"{name}: {full_waits} full wgmma waits for {mmas} MMAs (serialised pipeline)"


def test_conv_kernels_do_not_spill(res_usage):
    for name, r in res_usage.items():
        if _kernel(name) == "conv_tc_kernel":
            assert r["STACK"] == 0 and r["LOCAL"] == 0, f"{name}: {r['STACK']} B stack, {r['LOCAL']} B local memory (register spills)"
