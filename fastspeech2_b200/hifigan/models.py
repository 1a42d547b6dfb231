"""Drop-in `hifigan.models.Generator` (HiFi-GAN V1 generator): same constructor argument, checkpoint key layout
(weight_g / weight_v / bias), `remove_weight_norm()` and `forward(mel[B,80,T]) -> wav[B,1,256*T]` as the reference
(hifigan/models.py:112-174); forward is hand-written sm_90a CUDA behind fs2_vocoder_forward.  No PyTorch fallback.
"""
from __future__ import annotations

import contextlib
import ctypes as C

import torch
import torch.nn as nn

from .. import _lib as L
from .. import packing
from .._modtree import get, populate
from ..spec import hifigan_spec

LRELU_SLOPE = 0.1


def _cfg(h, name):
    return h[name] if isinstance(h, dict) else getattr(h, name)


class Generator(nn.Module):
    def __init__(self, h):
        super().__init__()
        self.h = h
        self._hd = {k: _cfg(h, k) for k in ("upsample_rates", "upsample_kernel_sizes", "upsample_initial_channel",
                                            "resblock_kernel_sizes", "resblock_dilation_sizes")}
        if str(_cfg(h, "resblock")) != "1":
            raise NotImplementedError("only resblock type '1' (HiFi-GAN V1, the shipped config) is supported")
        self.num_kernels = len(self._hd["resblock_kernel_sizes"])
        self.num_upsamples = len(self._hd["upsample_rates"])
        self._weight_norm = True
        self.use_tensor_cores = True     # split-FP16 tensor-core kernel for every conv it supports; False = fp32 CUDA-core kernels only
        # Operand split per part (bit 0 = conv_pre, bit 1+i = upsample stage i): set = fp16 main term + one E4M3 correction MMA
        # (half the tensor-core work of the three-MMA split), clear = three fp16 MMAs.  Default: every upsample stage, NOT conv_pre --
        # its input is the raw log-mel (|x| up to 11.5), where the E4M3 correction of the shipped universal checkpoint misses the 1e-4
        # waveform bar (tests/test_gpu_model.py::test_hifigan_real_checkpoint_vs_reference; CPU emulation: scripts/emul_split_precision.py).
        self.f8_mask = 0b11110
        # Stages (bit i) whose ResBlock group runs as ONE persistent kernel with every intermediate on chip (fs2_resstack, available for
        # the 64- and 32-channel stages; those stages use the f16 + f8 operand format regardless of f8_mask).  Default: the 32-channel
        # stage, the most memory-bound one; the 64-channel stage stays on the per-layer path unless fused_mask |= 0b0100.
        self.fused_mask = 0b1000
        # Stages (bit i) where every (dilated conv, conv, +x) pair with kernel size <= pair_kmax runs as ONE fs2_resstack launch, so
        # that the intermediate never leaves the SM: worthwhile for the memory-bound k = 3 pairs of the 64-channel stage, while the
        # longer kernels are tensor-bound and keep their per-layer launches -- hence pair_kmax = 3.
        self.pair_mask = 0b0100
        self.pair_kmax = 3
        populate(self, hifigan_spec(self._hd, weight_norm=True))
        with torch.no_grad():  # g = ||v|| so that the initial folded weight equals v, as torch's weight_norm does
            for base in self._bases():
                v = get(self, base + ".weight_v")
                get(self, base + ".weight_g").copy_(v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1))))
        self._packed = None
        self._ws = None

    # ------------------------------------------------------------------ weight-norm handling
    def _bases(self):
        seen = []
        for p in hifigan_spec(self._hd, weight_norm=False):
            if p.key.endswith(".weight"):
                seen.append(p.key[: -len(".weight")])
        return seen

    def _folded(self, base):
        if not self._weight_norm:
            return get(self, base + ".weight").detach()
        return packing.fold_weight_norm(get(self, base + ".weight_v").detach(), get(self, base + ".weight_g").detach())

    def remove_weight_norm(self):
        """Fold w = g * v/||v|| into plain `.weight` parameters (hifigan/models.py:167-174, :105-109)."""
        print("Removing weight norm...")
        if not self._weight_norm:
            raise ValueError("weight norm already removed")
        for base in self._bases():
            mod = self
            for name in base.split("."):
                mod = mod._modules[name]
            w = self._folded(base)
            del mod._parameters["weight_g"], mod._parameters["weight_v"]
            mod.register_parameter("weight", nn.Parameter(w))
        self._weight_norm = False
        self._invalidate()

    def _invalidate(self):
        self._packed = None
        self._ws = None

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self._invalidate()
        return out

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._invalidate()
        return out

    # ------------------------------------------------------------------ packing
    def _pack(self):
        L.lib()
        hd = self._hd
        dev = get(self, "conv_pre.bias").device
        if dev.type != "cuda":
            raise L.Fs2Error("hifigan.Generator (H100-native) needs its parameters on a CUDA device; there is no CPU path")
        m = L.VocoderModel()
        m.n_mel, m.c0 = 80, hd["upsample_initial_channel"]
        m.n_stages, m.n_kernels = self.num_upsamples, self.num_kernels
        m.n_dil = len(hd["resblock_dilation_sizes"][0])
        if m.n_stages > L.MAX_STAGES or m.n_stages * m.n_kernels > L.MAX_RESBLOCKS or m.n_dil > L.MAX_DIL or m.n_kernels > L.MAX_DIL + 4:
            raise L.Fs2Error("generator configuration exceeds the C ABI's fixed table sizes")
        for j, (k, dils) in enumerate(zip(hd["resblock_kernel_sizes"], hd["resblock_dilation_sizes"])):
            if len(dils) != m.n_dil:
                raise L.Fs2Error("ragged resblock_dilation_sizes unsupported")
            m.rb_k[j] = k
            for d, dv in enumerate(dils):
                m.rb_dil[j][d] = dv
        for i, (u, k) in enumerate(zip(hd["upsample_rates"], hd["upsample_kernel_sizes"])):
            if k != 2 * u or u % 2:
                raise L.Fs2Error("ConvTranspose1d stage needs kernel = 2*stride and even stride on the sm_90a path")
            m.rates[i], m.up_k[i] = u, k
        m.fused_mask = 0
        if self.use_tensor_cores:
            ch = m.c0
            for i in range(m.n_stages):
                ch //= 2
                if (int(self.fused_mask) >> i) & 1 and ch in (32, 64):
                    m.fused_mask |= 1 << i
        m.pair_mask, m.pair_kmax = (int(self.pair_mask) & ~m.fused_mask, int(self.pair_kmax)) if self.use_tensor_cores else (0, 0)
        m.f8_mask = (int(self.f8_mask) | (m.fused_mask << 1) | (m.pair_mask << 1)) if self.use_tensor_cores else 0
        pk = packing.pack_vocoder(lambda b: self._folded(b).float(), lambda b: get(self, b + ".bias").detach().float(),
                                  hd["upsample_rates"], m.n_stages * m.n_kernels, m.n_dil, f8_mask=m.f8_mask)
        P = lambda k: pk[k].data_ptr()
        m.w_pre, m.b_pre, m.w_post, m.b_post = P("w_pre"), P("b_pre"), P("w_post"), P("b_post")
        T = lambda k: pk[k + "_tc"].data_ptr() if (self.use_tensor_cores and k + "_tc" in pk) else 0
        m.w_pre_tc = T("w_pre")
        for i in range(m.n_stages):
            m.w_up_a[i], m.w_up_b[i], m.b_up[i] = P(f"up.{i}.wa"), P(f"up.{i}.wb"), P(f"up.{i}.b")
            m.w_up_a_tc[i], m.w_up_b_tc[i] = T(f"up.{i}.wa"), T(f"up.{i}.wb")
        for rb in range(m.n_stages * m.n_kernels):
            for d in range(m.n_dil):
                m.w_rb1[rb][d], m.b_rb1[rb][d] = P(f"rb.{rb}.{d}.w1"), P(f"rb.{rb}.{d}.b1")
                m.w_rb2[rb][d], m.b_rb2[rb][d] = P(f"rb.{rb}.{d}.w2"), P(f"rb.{rb}.{d}.b2")
                m.w_rb1_tc[rb][d], m.w_rb2_tc[rb][d] = T(f"rb.{rb}.{d}.w1"), T(f"rb.{rb}.{d}.w2")
        up = 1
        for u in hd["upsample_rates"]:
            up *= u
        self._packed = (m, pk, dev, up)
        return self._packed

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x, mel_lens=None):
        """x: mel [B, 80, T] (any strides; the usual caller passes postnet_mel.transpose(1, 2), utils/tools.py:202).

        mel_lens (optional): integer tensor [B] of valid frames per utterance, on any device (FastSpeech2's out[9] can be passed
        straight in).  Utterance b is then synthesised exactly as `self(x[b:b+1, :, :mel_lens[b]])` would synthesise it alone: frames
        at or beyond mel_lens[b] are never read, the vocoder skips the work of the padding, and wav[b, 0, t] = 0 for
        t >= mel_lens[b] * prod(upsample_rates).  The output shape stays [B, 1, prod(upsample_rates) * T].  Without mel_lens every
        utterance is synthesised over all T frames, padding included, as the reference does.  A CPU tensor is range-checked
        (ValueError outside [0, T]); device values are clamped to [0, T] by the kernels."""
        dev = get(self, "conv_pre.bias").device
        with (torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()):   # per-device kernel setup: CURRENT device
            return self._forward(x, mel_lens)

    def _forward(self, x, mel_lens=None):
        if self.training:
            raise NotImplementedError("H100-native hifigan.Generator is inference-only: call .eval() (utils/model.py:67)")
        lib = L.lib()
        m, _keep, dev, up = self._packed or self._pack()
        if x.dim() != 3 or x.shape[1] != m.n_mel:
            raise ValueError(f"expected mel of shape [B, {m.n_mel}, T]")
        x = x.to(device=dev, dtype=torch.float32)
        B, _, T = x.shape
        lens_d = None
        if mel_lens is not None:
            mel_lens = torch.as_tensor(mel_lens)
            if mel_lens.dtype.is_floating_point or mel_lens.dtype.is_complex or mel_lens.dtype == torch.bool or mel_lens.shape != (B,):
                raise ValueError(f"mel_lens must be an integer tensor of shape [{B}]")
            if mel_lens.device.type == "cpu" and B and not bool(((mel_lens >= 0) & (mel_lens <= T)).all()):
                raise ValueError(f"mel_lens must lie in [0, {T}]")
            lens_d = mel_lens.to(device=dev, dtype=torch.int32).contiguous()
        stream = torch.cuda.current_stream(dev).cuda_stream
        if x.stride(1) == 1 and x.stride(2) % 4 == 0 and x.stride(0) % 4 == 0 and x.data_ptr() % 16 == 0 and x.stride(2) >= m.n_mel:
            mel_cl, bs, rs = x, x.stride(0), x.stride(2)       # already a channels-last view
        else:
            xc = x.contiguous()
            mel_cl = torch.empty(B, T, m.n_mel, dtype=torch.float32, device=dev)
            L.check(lib.fs2_transpose_bct_to_btc(xc.data_ptr(), mel_cl.data_ptr(), B, m.n_mel, T, stream), "fs2_transpose")
            bs, rs = T * m.n_mel, m.n_mel
        wav = torch.empty(B, 1, T * up, dtype=torch.float32, device=dev)
        need = lib.fs2_vocoder_workspace_bytes(C.byref(m), B, T)
        if self._ws is None or self._ws.numel() < need or self._ws.device != dev:
            self._ws = torch.empty(need + 1024, dtype=torch.uint8, device=dev)
        va = L.VocoderArgs(B=B, T=T, mel=mel_cl.data_ptr(), mel_batch_stride=bs, mel_row_stride=rs, wav=wav.data_ptr(),
                           workspace=self._ws.data_ptr(), workspace_bytes=self._ws.numel(), mel_lens=L.ptr(lens_d))
        L.check(lib.fs2_vocoder_forward(C.byref(m), C.byref(va), stream), "fs2_vocoder_forward")
        return wav
