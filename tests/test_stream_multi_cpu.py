"""Streams of several generators in one vocoder pool, without a GPU: the C ABI of fs2_vocoder_forward_streams_multi (layout, host
checks, workspace), the pool's bookkeeping with a substituted launch call, and the SASS of the multi-generator entry points."""
import ctypes
import re

import pytest
import torch

from fastspeech2_b200 import _lib as L, configs
from fastspeech2_b200.hifigan import AttrDict, Generator
from fastspeech2_b200.hifigan.models import StreamPool
from tests.test_stream_open_cpu import _c_layout
from tests.test_stream_vocoder_cpu import _model


def test_abi_against_the_header():
    fields, csize = _c_layout("fs2_vocoder_streams_multi_args")
    cls = L.VocoderStreamsMultiArgs
    assert csize == ctypes.sizeof(cls) == L.VOCODER_STREAMS_MULTI_ARGS_SIZE == 88
    assert fields == [(n, getattr(cls, n).offset) for n, _ in cls._fields_]
    assert cls._fields_[:len(L.VocoderStreamsRingArgs._fields_)] == L.VocoderStreamsRingArgs._fields_
    header = open(re.sub(r"tests/.*", "include/fs2b200.h", __file__)).read()
    assert int(re.search(r"#define FS2_MAX_GENERATORS (\d+)", header).group(1)) == L.MAX_GENERATORS


def _models(n, cfg=configs.HIFIGAN_CONFIG, policy="default"):
    ms = [_model(cfg, policy)[0] for _ in range(n)]
    return ms, L.model_array(ms)


def test_workspace_is_the_streams_bound_plus_the_generator_table():
    h = L.lib()
    for cfg in (configs.HIFIGAN_CONFIG, configs.HIFIGAN_V2_CONFIG):
        for B in (1, 7, 64):
            ms, arr = _models(3, cfg)
            one = h.fs2_vocoder_streams_workspace_bytes(ctypes.byref(ms[0]), B, 32)
            multi = h.fs2_vocoder_streams_multi_workspace_bytes(arr, 3, B, 32)
            assert one < multi <= one + 4 * B + 256
            assert h.fs2_vocoder_streams_multi_workspace_bytes(arr, 1, B, 32) == multi
    ms, arr = _models(2)
    for n, B, frames in ((0, 4, 32), (L.MAX_GENERATORS + 1, 4, 32), (2, 0, 32), (2, 4, 0)):
        assert h.fs2_vocoder_streams_multi_workspace_bytes(arr, n, B, frames) == 0
    ms[1].c0 = 256
    assert h.fs2_vocoder_streams_multi_workspace_bytes(arr, 2, 4, 32) == 0


def _mismatches():
    """(what, edit of generator 1's struct) that the call must refuse"""
    def setp(name, value, idx=None):
        def f(m):
            if idx is None:
                setattr(m, name, value)
            else:
                arr = getattr(m, name)
                for i in idx[:-1]:
                    arr = arr[i]
                arr[idx[-1]] = value
        return f
    return [("c0", setp("c0", 256)), ("n_mel", setp("n_mel", 84)), ("rates", setp("rates", 10, (0,))),
            ("up_k", setp("up_k", 20, (1,))), ("rb_k", setp("rb_k", 5, (0,))), ("rb_dil", setp("rb_dil", 2, (1, 2))),
            ("f8_mask", setp("f8_mask", 0)), ("fused_mask", setp("fused_mask", 0b1000)), ("pair_mask", setp("pair_mask", 0b0010)),
            ("pair_kmax", setp("pair_kmax", 5)), ("w_pre_tc present", setp("w_pre_tc", 0x10000)),
            ("w_rb1_tc present", setp("w_rb1_tc", 0x10000, (3, 1))), ("b_up present", setp("b_up", 0x10000, (2,))),
            ("w_post present", setp("w_post", 0x10000))]


def test_multi_call_refuses_bad_arguments_before_any_cuda_call():
    h = L.lib()
    frames = 8
    ms, arr = _models(2)
    up = _model(configs.HIFIGAN_CONFIG)[1]
    need = h.fs2_vocoder_streams_multi_workspace_bytes(arr, 2, 2, frames)
    good = dict(B=2, frames=frames, mel=0x1000, mel_lens=0x1000, f0=0x1000, wav=0x1000, wav_batch_stride=frames * up,
                workspace=0x1000, workspace_bytes=need, cap=0, gen=0x1000, models_dev=0x1000)
    for k, v in (("B", 0), ("B", -1), ("frames", 0), ("mel", 0), ("mel_lens", 0), ("f0", 0), ("wav", 0), ("workspace", 0),
                 ("workspace_bytes", need - 1), ("wav_batch_stride", frames * up - 1), ("gen", 0), ("models_dev", 0)):
        a = L.VocoderStreamsMultiArgs(**dict(good, **{k: v}))
        assert h.fs2_vocoder_forward_streams_multi(arr, 2, ctypes.byref(a), None) == -1, (k, v)
    a = L.VocoderStreamsMultiArgs(**good)
    assert h.fs2_vocoder_forward_streams_multi(arr, 2, None, None) == -1
    assert h.fs2_vocoder_forward_streams_multi(None, 2, ctypes.byref(a), None) == -1
    for n in (0, -1, L.MAX_GENERATORS + 1):
        assert h.fs2_vocoder_forward_streams_multi(arr, n, ctypes.byref(a), None) == -1, n
    holed = (ctypes.POINTER(L.VocoderModel) * 2)(ctypes.pointer(ms[0]), ctypes.POINTER(L.VocoderModel)())   # a NULL model
    assert h.fs2_vocoder_forward_streams_multi(holed, 2, ctypes.byref(a), None) == -1
    for what, edit in _mismatches():
        bad, bad_arr = _models(2)
        edit(bad[1])
        assert h.fs2_vocoder_forward_streams_multi(bad_arr, 2, ctypes.byref(a), None) == -1, what
    # the same pointer present at another address modulo 16 is another weight format
    m0, m1 = _model(configs.HIFIGAN_CONFIG)[0], _model(configs.HIFIGAN_CONFIG)[0]
    m0.w_post, m1.w_post = 0x10000, 0x10008
    assert h.fs2_vocoder_forward_streams_multi(L.model_array([m0, m1]), 2, ctypes.byref(a), None) == -1


class _Launch:
    """A substituted launch call that records its arguments: a [B, chunk * up] zero waveform per call."""

    def __init__(self, up, chunk):
        self.up, self.chunk, self.calls = up, chunk, []

    def __call__(self, ptrs, f0s, ns, caps=None, gens=None):
        self.calls.append(dict(ptrs=list(ptrs), f0s=list(f0s), ns=list(ns), caps=caps, gens=gens))
        return torch.zeros(len(ptrs), self.chunk * self.up)


def test_generator_indices_reach_the_launch_in_admission_order():
    up, chunk = 4, 2
    launch = _Launch(up, chunk)
    pool = StreamPool(launch, 80, up, chunk, "cpu", append=lambda records: None, n_generators=3)
    lens_gens = [(5, 2), (3, 0), (6, 1), (2, 2)]
    handles = [pool.add(torch.zeros(80, n), generator=g) for n, g in lens_gens]
    h_open = pool.open(generator=1)
    pool.feed(h_open, torch.zeros(80, 40))
    pool.close(h_open)
    steps = 0
    while len(pool):
        out = pool.step()
        steps += 1
        assert len(launch.calls) == steps                  # one call per step whatever the mix
        call = launch.calls[-1]
        live = [h for h, _, _ in out]
        expect = [dict(zip(handles + [h_open], [g for _, g in lens_gens] + [1]))[h] for h in live]
        assert call["gens"] == expect
        assert live == sorted(live)                         # admission order
    assert launch.calls[0]["gens"] == [2, 0, 1, 2, 1]
    assert launch.calls[0]["caps"] is not None             # the open stream puts the step on rings


def test_one_generator_pool_calls_the_old_launch_signature():
    calls = []

    def launch(ptrs, f0s, ns, caps=None):                  # no gens keyword: a one-generator pool must not pass one
        calls.append(caps)
        return torch.zeros(len(ptrs), 8)

    pool = StreamPool(launch, 80, 4, 2, "cpu", append=lambda records: None)
    pool.add(torch.zeros(80, 3))
    pool.add(torch.zeros(80, 5), generator=0)
    while len(pool):
        pool.step()
    assert calls == [None, None, None]
    h = pool.open()
    pool.feed(h, torch.zeros(80, 4))
    pool.close(h)
    while len(pool):
        pool.step()
    assert calls[3] is not None


def test_generator_index_errors():
    pool = StreamPool(_Launch(4, 2), 80, 4, 2, "cpu", append=lambda records: None, n_generators=2)
    for g in (2, -1, True, 1.0, "0", None):
        with pytest.raises(ValueError):
            pool.add(torch.zeros(80, 3), generator=g)
        with pytest.raises(ValueError):
            pool.open(generator=g)
    assert len(pool) == 0
    one = StreamPool(_Launch(4, 2), 80, 4, 2, "cpu")
    with pytest.raises(ValueError):
        one.add(torch.zeros(80, 3), generator=1)


def _gen(cfg=configs.HIFIGAN_CONFIG, **attrs):
    g = Generator(AttrDict(cfg))
    g.eval()
    for k, v in attrs.items():
        setattr(g, k, v)
    return g


@pytest.mark.parametrize("other", [
    lambda: _gen(configs.HIFIGAN_V2_CONFIG),
    lambda: _gen(AttrDict(dict(configs.HIFIGAN_CONFIG, sampling_rate=24000))),
    lambda: _gen(AttrDict(dict(configs.HIFIGAN_CONFIG, resblock_dilation_sizes=[[1, 3, 5], [1, 3, 5], [1, 2, 5]]))),
    lambda: _gen(use_tensor_cores=False),
    lambda: _gen(fused_mask=0),
    lambda: _gen(wide_pairs=True),
    lambda: _gen(f8_mask=0b11111),
    lambda: _gen().train(),
    lambda: torch.nn.Linear(2, 2),
], ids=["v2", "rate", "dilations", "no_tc", "fused_mask", "wide_pairs", "f8_mask", "training", "not_a_generator"])
def test_pool_creation_refuses_a_generator_it_cannot_share_a_plan_with(other):
    with pytest.raises(ValueError):
        _gen().stream_pool(generators=(other(),))


def test_pool_creation_refuses_more_than_max_generators():
    g = _gen()
    with pytest.raises(ValueError):
        g.stream_pool(generators=tuple(_gen() for _ in range(L.MAX_GENERATORS)))


# --------------------------------------------------------------------------- SASS of the multi-generator entry points
# the table mode's windowed entry points (mangled-name patterns): conv_tc_table_kernel<NB, true, true> and the fused ResBlock ones
MULTI_KERNELS = {r"\dconv_tc_table_kernelILi\d+ELb1ELb1E": 8, r"\dresstack_multi_kernelI": 2, r"\dresstack_multi_narrow_kernelI": 2,
                 r"\dresstack_multi_wide_kernelE": 1}


def test_windowed_table_entry_points_are_pipelined_and_the_conv_does_not_spill():
    from tests.test_sass_pipeline import mmas_and_full_waits, res_usage_of, sass_of
    keep = re.compile("|".join(MULTI_KERNELS)).search
    sass, usage = sass_of(keep), res_usage_of(keep)
    for kernel, n in MULTI_KERNELS.items():
        names = [f for f in sass if re.search(kernel, f)]
        assert len(names) == n and sum(bool(re.search(kernel, f)) for f in usage) == n, kernel
        for f in names:
            mmas, full_waits = mmas_and_full_waits(sass[f])
            assert mmas > 0 and full_waits * 4 <= mmas, (f, mmas, full_waits)
            if "conv_tc_table_kernel" in kernel:
                assert usage[f]["STACK"] == 0 and usage[f]["LOCAL"] == 0, (f, usage[f])
