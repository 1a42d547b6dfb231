"""CPU: the windowed (streaming) vocoder's host side -- fs2_vocoder_window_plan, the workspace bound, the ABI of the new calls -- and its
receptive field against the CPU oracle.  The GPU side (bits of every window against forward) is tests/test_gpu_stream_vocoder.py."""
import ctypes

import pytest
import torch

from fastspeech2_b200 import _lib as L, configs, synth
from fastspeech2_b200.hifigan import AttrDict, Generator
from oracle import fs2_oracle as O

# V1, V2, and a generator with other kernel sizes, dilations and rates (a 6x stage, two dilations per ResBlock, kernel 9)
OTHER_CONFIG = dict(configs.HIFIGAN_CONFIG, upsample_rates=[6, 4, 2, 4], upsample_kernel_sizes=[12, 8, 4, 8], upsample_initial_channel=256,
                    resblock_kernel_sizes=[3, 5, 9], resblock_dilation_sizes=[[1, 2], [1, 3], [2, 4]])
CONFIGS = {"v1": configs.HIFIGAN_CONFIG, "v2": configs.HIFIGAN_V2_CONFIG, "other": OTHER_CONFIG}
# (use_tensor_cores, fused_mask, pair_mask): the defaults, pairs instead of fused groups, per-layer convs only, no tensor cores
POLICIES = {"default": (True, None, None), "pairs": (True, 0, 0b1111), "per_layer": (True, 0, 0), "exact": (False, None, None)}


def _model(cfg, policy="default"):
    """The fs2_vocoder_model the Generator would pack (only the shape fields and masks: the plan reads no pointer)."""
    h = AttrDict(cfg)
    gen = Generator(h)
    tc, fused, pair = POLICIES[policy]
    gen.use_tensor_cores = tc
    if fused is not None:
        gen.fused_mask, gen.pair_mask = fused, pair
    m = L.VocoderModel()
    m.n_mel, m.c0 = 80, h.upsample_initial_channel
    m.n_stages, m.n_kernels, m.n_dil = len(h.upsample_rates), len(h.resblock_kernel_sizes), len(h.resblock_dilation_sizes[0])
    for i, (u, k) in enumerate(zip(h.upsample_rates, h.upsample_kernel_sizes)):
        m.rates[i], m.up_k[i] = u, k
    for j, (k, dils) in enumerate(zip(h.resblock_kernel_sizes, h.resblock_dilation_sizes)):
        m.rb_k[j] = k
        for d, dv in enumerate(dils):
            m.rb_dil[j][d] = dv
    m.f8_mask, m.fused_mask, m.pair_mask, m.pair_kmax = gen.effective_masks()
    up = 1
    for u in h.upsample_rates:
        up *= u
    return m, up


def _windows(T):
    return [(0, 16), (0, 1), (T // 3, T // 3 + 21), (T - 16, T), (T - 5, T + 40), (T - 1, T), (T // 2, T // 2 + 1), (0, T + 7)]


def _check_plan(m, up, T, f0, f1):
    P = L.vocoder_window_plan(m, T, f0, f1)
    assert P[0].layer == L.VW_CONV_PRE and P[-1].layer == L.VW_CONV_POST
    assert (P[-1].y0, P[-1].y1) == (f0 * up, min(f1, T) * up)
    for i, l in enumerate(P):
        cap = T * l.scale
        assert 0 <= l.y0 < l.y1 <= cap and 0 <= l.x0 < l.x1 <= cap, (i, l.layer)
        if l.src < 0:
            assert l.layer == L.VW_CONV_PRE and l.scale == 1
        else:
            assert l.src < i
            p = P[l.src]
            f = l.scale // p.scale                            # a ConvTranspose group's row q holds the next rate's rows [q*u, q*u + u)
            assert f * p.scale == l.scale
            assert p.y0 * f <= l.x0 and l.x1 <= min(p.y1 * f, cap), (i, l.layer, (l.x0, l.x1), (p.y0 * f, p.y1 * f))
        if l.res_src >= 0:
            p = P[l.res_src]
            f = l.scale // p.scale
            assert p.y0 * f <= l.y0 and l.y1 <= p.y1 * f, (i, l.layer)
    return P


@pytest.mark.parametrize("policy", list(POLICIES))
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_every_launch_reads_inside_its_producers_rows(cfg, policy):
    m, up = _model(CONFIGS[cfg], policy)
    for T in (1, 5, 40, 101):
        for f0, f1 in _windows(T):
            if 0 <= f0 < T and f1 > f0:
                _check_plan(m, up, T, f0, f1)


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_launches_follow_the_masks(cfg):
    m, _ = _model(CONFIGS[cfg])
    kinds = {l.layer for l in L.vocoder_window_plan(m, 50, 10, 20)}
    assert (L.VW_RB_GROUP in kinds) == (m.fused_mask != 0)
    assert L.VW_RB_GROUP not in {l.layer for l in L.vocoder_window_plan(_model(CONFIGS[cfg], "per_layer")[0], 50, 10, 20)}


@pytest.mark.parametrize("chunk", [1, 7, 64, 200])
@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_consecutive_windows_tile_the_waveform(cfg, chunk):
    m, up = _model(CONFIGS[cfg])
    T = 150
    edges = [L.vocoder_window_plan(m, T, f0, f0 + chunk)[-1] for f0 in range(0, T, chunk)]
    assert edges[0].y0 == 0 and edges[-1].y1 == T * up
    assert all(a.y1 == b.y0 for a, b in zip(edges, edges[1:]))


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_workspace_is_bounded_by_the_window_not_by_T(cfg):
    m, up = _model(CONFIGS[cfg])
    h = L.lib()
    for B in (1, 3):
        ws = {fr: h.fs2_vocoder_window_workspace_bytes(ctypes.byref(m), B, fr) for fr in (1, 16, 64, 128)}
        assert 0 < ws[1] <= ws[16] <= ws[64] <= ws[128]
        # the five buffers hold every launch's output rows of any window of those frames, at any T and position
        for T in (64, 1000, 20000):
            for f0 in (0, T // 2, T - 64):
                for l in L.vocoder_window_plan(m, T, f0, f0 + 64):
                    if l.layer == L.VW_CONV_POST:
                        continue
                    ch = m.c0 if l.layer == L.VW_CONV_PRE else (m.c0 >> (l.stage + 1)) * (
                        m.rates[l.stage] if l.layer in (L.VW_UP_A, L.VW_UP_B) else 1)
                    assert 5 * B * (l.y1 - l.y0) * ch * 4 <= ws[64]
        full = h.fs2_vocoder_workspace_bytes(ctypes.byref(m), B, 20000)
        assert ws[64] * 50 < full


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_offline_workspace_is_five_buffers_of_the_widest_layer(cfg):
    """fs2_vocoder_workspace_bytes: five 256-byte aligned buffers of B * T * max(c0, max_i up_i * c_i) floats, with up_i the rows per
    mel frame after stage i and c_i = c0 >> (i + 1) its channels, plus 256 bytes."""
    m, _ = _model(CONFIGS[cfg])
    per_frame, up = m.c0, 1
    for i in range(m.n_stages):
        up *= m.rates[i]
        per_frame = max(per_frame, up * (m.c0 >> (i + 1)))
    for B in (1, 3, 16):
        for T in (1, 7, 127, 1011):
            n = 4 * B * T * per_frame
            assert L.lib().fs2_vocoder_workspace_bytes(ctypes.byref(m), B, T) == 4 * ((n + 255) // 256 * 256) + n + 256, (B, T)


def test_unsupported_models_are_refused_before_any_cuda_call():
    """A model the walk cannot run is refused by forward before its first launch (the pointers below are never dereferenced), and
    has no workspace size."""
    h = L.lib()
    T = 40
    a = L.VocoderArgs(B=2, T=T, mel=0x1000, mel_batch_stride=T * 80, mel_row_stride=80, wav=0x1000, workspace=0x1000,
                      workspace_bytes=1 << 40)
    m, _ = _model(configs.HIFIGAN_CONFIG)
    m.up_k[2] = 2 * m.rates[2] + 2                     # the ConvTranspose runs as two 2-tap phase groups only at up_k = 2 * rate
    assert h.fs2_vocoder_workspace_bytes(ctypes.byref(m), 2, T) == 0
    assert h.fs2_vocoder_forward(ctypes.byref(m), ctypes.byref(a), None) == -2     # FS2_ERR_UNSUPPORTED
    m, _ = _model(configs.HIFIGAN_CONFIG)
    m.fused_mask, m.f8_mask = 0b1000, m.f8_mask & ~(2 << 3)   # a fused stage without its f16 + f8 tiles
    assert h.fs2_vocoder_workspace_bytes(ctypes.byref(m), 2, T) == 0
    assert h.fs2_vocoder_forward(ctypes.byref(m), ctypes.byref(a), None) == -1     # FS2_ERR_ARG


@pytest.mark.parametrize("cfg", ["v1", "v2"])
def test_streamed_work_is_within_ten_percent_of_offline(cfg):
    """Algorithmic FLOPs (every conv over the rows its consumers need) of a 1012-frame utterance in 64-frame chunks."""
    m, _ = _model(CONFIGS[cfg])
    T = 1012
    offline = sum(l.flops for l in L.vocoder_window_plan(m, T, 0, T))
    streamed = sum(l.flops for f0 in range(0, T, 64) for l in L.vocoder_window_plan(m, T, f0, f0 + 64))
    assert offline > 0 and streamed / offline <= 1.10, streamed / offline


def test_abi_of_the_window_calls():
    h = L.lib()
    assert h.fs2_abi_version() == L.ABI_VERSION == 12
    assert h.fs2_struct_size(19) == 0
    assert ctypes.sizeof(L.VocoderWindowArgs) == L.VOCODER_WINDOW_ARGS_SIZE == 80
    assert ctypes.sizeof(L.VocoderWindowLaunch) == L.VOCODER_WINDOW_LAUNCH_SIZE == 56
    # the fields of fs2_vocoder_args, in order, then the window
    assert [f[0] for f in L.VocoderWindowArgs._fields_][:9] == [f[0] for f in L.VocoderArgs._fields_]


def test_bad_windows_are_refused_before_any_cuda_call():
    h = L.lib()
    m, up = _model(configs.HIFIGAN_CONFIG)
    T = 40
    for f0, f1 in ((-1, 5), (5, 5), (6, 5), (T, T + 3), (T + 2, T + 9)):
        a = L.VocoderWindowArgs(B=2, T=T, mel=0x1000, mel_batch_stride=T * 80, mel_row_stride=80, wav=0x1000, workspace=0x1000,
                                workspace_bytes=1 << 40, f0=f0, f1=f1, wav_batch_stride=T * up)
        assert h.fs2_vocoder_forward_window(ctypes.byref(m), ctypes.byref(a), None) == -1, (f0, f1)
        assert h.fs2_vocoder_window_plan(ctypes.byref(m), T, f0, f1, None, 0) == -1, (f0, f1)
    a = L.VocoderWindowArgs(B=2, T=T, mel=0x1000, mel_batch_stride=T * 80, mel_row_stride=80, wav=0x1000, workspace=0x1000,
                            workspace_bytes=1 << 40, f0=0, f1=8, wav_batch_stride=8 * up - 1)   # chunks would overlap
    assert h.fs2_vocoder_forward_window(ctypes.byref(m), ctypes.byref(a), None) == -1
    assert h.fs2_vocoder_window_workspace_bytes(ctypes.byref(m), 2, 0) == 0


@pytest.mark.parametrize("cfg,T", [("v2", 48), ("v1", 30)])
def test_receptive_field_against_the_oracle(cfg, T):
    """Perturb mel frame j of the CPU oracle generator: every output sample that changes lies in a frame f whose one-frame window's
    plan reads j (conv_pre's input rows)."""
    h = AttrDict(CONFIGS[cfg])
    m, up = _model(CONFIGS[cfg])
    sd = synth.hifigan_state_dict(h, seed=4)
    kw = dict(upsample_rates=h.upsample_rates, upsample_kernel_sizes=h.upsample_kernel_sizes,
              resblock_kernel_sizes=h.resblock_kernel_sizes, resblock_dilation_sizes=h.resblock_dilation_sizes, dtype=torch.float64)
    mel = synth.make_mel(1, T, seed=5).double()
    base = O.hifigan_forward(sd, mel, **kw)[0, 0]
    reads = [L.vocoder_window_plan(m, T, f, f + 1)[0] for f in range(T)]
    for j in (0, T // 2, T - 1):
        mel2 = mel.clone()
        mel2[0, :, j] += 3.0
        changed = (O.hifigan_forward(sd, mel2, **kw)[0, 0] != base).nonzero().flatten()
        assert len(changed) > 0
        for f in sorted({int(s) // up for s in changed}):
            assert reads[f].x0 <= j < reads[f].x1, (j, f, reads[f].x0, reads[f].x1)


# The windowed mode's own entry points (conv_tc_streams_kernel, resstack_streams_kernel, resstack_narrow_streams_kernel), which the
# window and streams calls run, get the checks tests/test_sass_pipeline.py makes of the padded and ragged ones: pipelined wgmma groups,
# and no spills in the conv kernel.
WINDOW_KERNELS = {"conv_tc_streams_kernel": 8, "resstack_streams_kernel": 2, "resstack_narrow_streams_kernel": 2}


@pytest.fixture(scope="module")
def window_sass():
    import re
    import subprocess
    from tests.test_sass_pipeline import LIB, _cuobjdump
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    funcs, name = {}, None
    for line in subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in WINDOW_KERNELS) else None
            if name:
                funcs[name] = []
        elif name:
            funcs[name].append(line)
    usage, name = {}, None
    for line in subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1) if any(k in m.group(1) for k in WINDOW_KERNELS) else None
        elif name and "REG:" in line:
            usage[name] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
            name = None
    return {k: "\n".join(v) for k, v in funcs.items()}, usage


def test_windowed_entry_points_are_pipelined_and_the_conv_does_not_spill(window_sass):
    import re
    sass, usage = window_sass
    for kernel, n in WINDOW_KERNELS.items():
        names = [f for f in sass if re.search(r"\d" + kernel + "I", f)]
        assert len(names) == n and sum(bool(re.search(r"\d" + kernel + "I", f)) for f in usage) == n, kernel
        for f in names:
            mmas = len(re.findall(r"\b[HQ]GMMA\.", sass[f]))
            full_waits = len(re.findall(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x0\b", sass[f]))
            assert mmas > 0 and full_waits * 4 <= mmas, (f, mmas, full_waits)
            if kernel == "conv_tc_streams_kernel":
                assert usage[f]["STACK"] == 0 and usage[f]["LOCAL"] == 0, (f, usage[f])
