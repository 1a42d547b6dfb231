"""Drop-in `hifigan.models.Generator` (HiFi-GAN V1 and V2 generators): same constructor argument, checkpoint key layout
(weight_g / weight_v / bias), `remove_weight_norm()` and `forward(mel[B,80,T]) -> wav[B,1,256*T]` as the reference
(hifigan/models.py:112-174); forward is hand-written sm_90a CUDA behind fs2_vocoder_forward.  No PyTorch fallback.
"""
from __future__ import annotations

import collections
import contextlib
import ctypes as C

import numpy as np
import torch
import torch.nn as nn

from .. import _lib as L
from .. import _streams
from .. import ops, packing
from .._modtree import get, populate
from ..resample import ENCODINGS, Resampler
from ..spec import hifigan_spec

LRELU_SLOPE = 0.1


def _cfg(h, name):
    return h[name] if isinstance(h, dict) else getattr(h, name)


# Channel counts of the stages whose ResBlock group fs2_resstack runs as one launch
FUSED_WIDTHS = (8, 16, 32, 64)


class Generator(nn.Module):
    """HiFi-GAN generator for every `resblock: "1"` config the reference's Generator builds: V1 (upsample_initial_channel 512) and
    V2 (128).  `resblock: "2"` (V3) is not in the reference's Generator and stays NotImplementedError."""

    def __init__(self, h):
        super().__init__()
        self.h = h
        self._hd = {k: _cfg(h, k) for k in ("upsample_rates", "upsample_kernel_sizes", "upsample_initial_channel",
                                            "resblock_kernel_sizes", "resblock_dilation_sizes")}
        if str(_cfg(h, "resblock")) != "1":
            raise NotImplementedError("only resblock type '1' (HiFi-GAN V1 and V2) is supported")
        self.num_kernels = len(self._hd["resblock_kernel_sizes"])
        self.num_upsamples = len(self._hd["upsample_rates"])
        self._weight_norm = True
        self.use_tensor_cores = True     # split-FP16 tensor-core kernel for every conv it supports; False = fp32 CUDA-core kernels only
        # Operand split per part (bit 0 = conv_pre, bit 1+i = upsample stage i): set = fp16 main term + one E4M3 correction MMA
        # (half the tensor-core work of the three-MMA split), clear = three fp16 MMAs.  Default: every upsample stage, NOT conv_pre --
        # its input is the raw log-mel (|x| up to 11.5), where the E4M3 correction of the shipped universal checkpoint misses the 1e-4
        # waveform bar (tests/test_gpu_model.py::test_hifigan_real_checkpoint_vs_reference; CPU emulation: scripts/emul_split_precision.py).
        self.f8_mask = 0b11110
        # Stages (bit i) whose ResBlock group runs on the persistent fs2_resstack kernel with the intermediates of each launch on chip
        # (available for the 64-, 32-, 16- and 8-channel stages; those stages use the f16 + f8 operand format regardless of f8_mask).
        # The library cuts such a stage into the whole group or runs of each ResBlock's dilations, whichever its cost model of halo
        # recompute rates fastest (fs2_vocoder_resblock_runs); every cut gives the same bits.  Default: every
        # stage it serves, 0b1100 for V1 (on an H100 SXM at 400 W, bench.py configs[2]: 127 ms per step against 133 ms with the
        # 64-channel stage on per-layer launches and fused k = 3 pairs) and 0b1111 for V2.
        self.fused_mask = self._fusable_stages()
        # Stages (bit i) where every (dilated conv, conv, +x) pair with kernel size <= pair_kmax runs as ONE fs2_resstack launch, so
        # that the intermediate never leaves the SM.  Only stages outside fused_mask use it: by default none.  Bit 2 is V1's 64-channel
        # stage (its memory-bound k = 3 pairs when that stage is taken out of fused_mask) and V2's 16-channel stage, so with
        # fused_mask = 0 V2 still pairs that stage; clear pair_mask too for all-per-layer ResBlocks.
        self.pair_mask = 0b0100
        self.pair_kmax = 3
        # The 128-channel stage (V1's second) too runs its pairs with kernel size <= pair_kmax as fs2_resstack launches (pair_mask bit
        # 8 + i of the C ABI; its f16 + f8 tiles are then packed at 128 output channels per block).  Bit-identical to the per-layer
        # convs, three launches instead of six; off by default (DESIGN.md section 5: 69.4 -> 68.1 ms for V1 at B = 16 x 1012).
        self.wide_pairs = False
        populate(self, hifigan_spec(self._hd, weight_norm=True))
        with torch.no_grad():  # g = ||v|| so that the initial folded weight equals v, as torch's weight_norm does
            for base in self._bases():
                v = get(self, base + ".weight_v")
                get(self, base + ".weight_g").copy_(v.reshape(v.shape[0], -1).norm(dim=1).reshape(-1, *([1] * (v.dim() - 1))))
        self._packed = None
        self._packed_state = None      # _streams.StreamState of the packed weights: made on the stream of the call that packed them
        self._ws, self._ws_stream = None, None     # the last forward's workspace and the stream it was allocated on (_streams.workspace)

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
        if self._packed is not None:
            self._packed_state.release(*self._packed[1].values())
        self._packed = None
        self._ws = self._ws_stream = None

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self._invalidate()
        return out

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._invalidate()
        return out

    # ------------------------------------------------------------------ packing
    def _fusable_stages(self):
        """Bit i set when stage i's width (upsample_initial_channel / 2^(i+1)) is one fs2_resstack serves."""
        return self._stages_of_width(*FUSED_WIDTHS)

    def _stages_of_width(self, *widths):
        mask, ch = 0, self._hd["upsample_initial_channel"]
        for i in range(self.num_upsamples):
            ch //= 2
            if ch in widths:
                mask |= 1 << i
        return mask

    def effective_masks(self):
        """(f8_mask, fused_mask, pair_mask, pair_kmax) as the C ABI receives them (fs2_vocoder_model): fusion only for the
        stages whose width fs2_resstack serves (FUSED_WIDTHS), pairs only outside the fused stages, and every fused or paired
        stage in the f16 + f8 format.  All zero without tensor cores."""
        if not self.use_tensor_cores:
            return 0, 0, 0, 0
        fused = int(self.fused_mask) & self._fusable_stages()
        pair = int(self.pair_mask) & ~fused
        wide = self._stages_of_width(128) if self.wide_pairs else 0
        return int(self.f8_mask) | (fused << 1) | (pair << 1) | (wide << 1), fused, pair | (wide << 8), int(self.pair_kmax)

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
        m.f8_mask, m.fused_mask, m.pair_mask, m.pair_kmax = self.effective_masks()
        wide_keys = [f"rb.{i * m.n_kernels + j}.{d}.{w}" for i in range(m.n_stages) if (m.pair_mask >> (8 + i)) & 1
                     for j in range(m.n_kernels) if m.rb_k[j] <= m.pair_kmax for d in range(m.n_dil) for w in ("w1", "w2")]
        pk = packing.pack_vocoder(lambda b: self._folded(b).float(), lambda b: get(self, b + ".bias").detach().float(),
                                  hd["upsample_rates"], m.n_stages * m.n_kernels, m.n_dil, f8_mask=m.f8_mask,
                                  wide_keys=wide_keys if self.use_tensor_cores else ())
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
        self._packed_state = _streams.made(dev)
        return self._packed

    def _packed_on_stream(self):
        """_packed (packing it first if needed), ready on the current stream."""
        packed = self._packed or self._pack()
        self._packed_state.enter()
        return packed

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, x, mel_lens=None):
        """x: mel [B, 80, T] (any strides; the usual caller passes postnet_mel.transpose(1, 2), utils/tools.py:202).

        mel_lens (optional): integer tensor [B] of valid frames per utterance, on any device (FastSpeech2's out[9] can be passed
        straight in).  Utterance b is then synthesised exactly as `self(x[b:b+1, :, :mel_lens[b]])` would synthesise it alone: frames
        at or beyond mel_lens[b] are never read, the vocoder skips the work of the padding, and wav[b, 0, t] = 0 for
        t >= mel_lens[b] * prod(upsample_rates).  The output shape stays [B, 1, prod(upsample_rates) * T].  Without mel_lens every
        utterance is synthesised over all T frames, padding included, as the reference does.  A CPU tensor is range-checked
        (ValueError outside [0, T]); device values are clamped to [0, T] by the kernels.

        CUDA streams: the call enqueues all of its device work on the stream current at the call.  Its workspace is cached for the next
        call on the same stream only: a call on another stream allocates its own, so calls on two streams never share one.  x, mel_lens
        and the returned waveform follow torch's usual rule: the caller orders them across streams.  The weights packed by the first
        call are ready on whatever stream a later call uses, and are not freed while another stream's queued work reads them."""
        dev = get(self, "conv_pre.bias").device
        with (torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()):   # per-device kernel setup: CURRENT device
            return self._forward(x, mel_lens)

    def _inputs(self, x, mel_lens):
        """Checks the arguments of forward / stream and converts them once: (model, packed weights, device, up, B, T, channels-last mel
        view, its batch and row strides, device mel_lens or None, stream)."""
        if self.training:
            raise NotImplementedError("H100-native hifigan.Generator is inference-only: call .eval() (utils/model.py:67)")
        lib = L.lib()
        m, keep, dev, up = self._packed_on_stream()
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
        return m, keep, dev, up, B, T, mel_cl, bs, rs, lens_d, stream

    def _forward(self, x, mel_lens=None):
        lib = L.lib()
        m, _keep, dev, up, B, T, mel_cl, bs, rs, lens_d, stream = self._inputs(x, mel_lens)
        wav = torch.empty(B, 1, T * up, dtype=torch.float32, device=dev)
        self._ws, self._ws_stream = _streams.workspace((self._ws, self._ws_stream), lib.fs2_vocoder_workspace_bytes(C.byref(m), B, T),
                                                       dev, slack=1024)
        ws = self._ws
        va = L.VocoderArgs(B=B, T=T, mel=mel_cl.data_ptr(), mel_batch_stride=bs, mel_row_stride=rs, wav=wav.data_ptr(),
                           workspace=ws.data_ptr(), workspace_bytes=ws.numel(), mel_lens=L.ptr(lens_d))
        L.check(lib.fs2_vocoder_forward(C.byref(m), C.byref(va), stream), "fs2_vocoder_forward")
        return wav

    @torch.no_grad()
    def stream(self, x, mel_lens=None, chunk_frames=64, sample_rate=None, pcm16=False):
        """Synthesise in chunks of `chunk_frames` mel frames: an iterator of (first_sample, wav_chunk[B, 1, n]), the chunks in order,
        whose concatenation along the last axis equals forward(x, mel_lens) bit for bit (fs2_vocoder_forward_window).  Each chunk is
        computed from the frames it needs plus the generator's receptive field, in a workspace that depends on B and chunk_frames, not
        on T, and is ready as soon as it is yielded (on the current stream), before the rest of the utterance is synthesised.  The
        arguments are those of forward and are checked, and the mel converted, once, when stream() is called; device mel_lens are
        never read on the host, so every utterance runs the batch's T frames in lockstep (chunks past an utterance's end are zeros).

        sample_rate (optional): yield the waveform at this rate instead of h.sampling_rate (resample.Resampler): one chunk per vocoder
        chunk, holding the outputs whose support has arrived (the last chunk flushes the rest), with first_sample at the new rate.
        Concatenated, they equal Resampler(h.sampling_rate, sample_rate)(forward(x, mel_lens), mel_lens * hop) bit for bit, hop =
        prod(upsample_rates) (without mel_lens: of forward(x)); pcm16 yields that output's int16 conversion (x 32768, truncated,
        clamped).  The lag behind the vocoder is about half_len / up input samples, under 1 ms at 8 to 48 kHz.

        CUDA streams: stream() enqueues the mel's conversion on the stream current when it is called, and each next() enqueues its
        chunk on the stream current at that next(), after the iterator's earlier work on any other stream (converted mel, previous
        chunk), with no host sync.  x, mel_lens and the yielded chunks follow torch's usual rule: the caller orders them across
        streams.  The iterator's own tensors are not freed while a stream it ran on still has queued work that reads them."""
        if isinstance(chunk_frames, bool) or not isinstance(chunk_frames, int) or chunk_frames < 1:
            raise ValueError("chunk_frames must be a positive int")
        rs = self._resampler(sample_rate, chunk_frames)
        dev = get(self, "conv_pre.bias").device
        with (torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()):
            inputs = self._inputs(x, mel_lens)
            state = _streams.made(dev)             # the iterator's last enqueued work: the mel's conversion, then each chunk
        if rs is None and not pcm16:
            return self._stream(inputs, chunk_frames, state)
        return self._stream_resampled(inputs, chunk_frames, rs, pcm16, state)

    def _resampler(self, sample_rate, chunk_frames):
        """The Resampler from h.sampling_rate to sample_rate, or None (sample_rate None or equal).  A window needs Resampler.history
        input samples before its first output's support, which the previous chunk must hold: ValueError otherwise."""
        if sample_rate is None:
            return None
        rs = Resampler(_cfg(self.h, "sampling_rate"), sample_rate)
        if rs.identity:
            return None
        hop = int(np.prod(self._hd["upsample_rates"]))
        if chunk_frames * hop < rs.history:
            raise ValueError(f"chunk_frames * {hop} samples must cover the resampler's history of {rs.history} samples")
        return rs

    def _stream_resampled(self, inputs, chunk_frames, rs, pcm16, state):
        _m, _keep, dev, up, B, T, _mel, _bs, _rs, lens_d, _ = inputs
        N = T * up
        prev, emitted = None, 0
        with torch.no_grad(), torch.cuda.device(dev):
            # _stream enters the iterator's state before each chunk; the chunk's conversion is recorded here, before it is yielded
            for i1, wav in self._stream(inputs, chunk_frames, state, record=False):  # i1: the chunk's first sample
                cur = wav[:, 0]
                if rs is None:                                  # the generator's own rate, int16 (samples past mel_lens are zeros)
                    y = ops.wav_to_int16(cur)
                    state.record()
                    yield i1, y.unsqueeze(1)
                    continue
                i2 = i1 + cur.shape[1]
                r = rs.ready(i2, N, i2 >= N)
                if r > emitted:
                    y = rs.window(prev, cur, i1, N, emitted, r, lens=lens_d, lens_scale=up, pcm16=pcm16)
                else:
                    y = torch.empty(B, 0, dtype=torch.int16 if pcm16 else torch.float32, device=dev)
                state.record()
                state.release(prev)
                j0, prev, emitted = emitted, cur, r
                yield j0, y.unsqueeze(1)

    def _stream(self, inputs, chunk_frames, state, record=True):
        """The chunks of stream(): each enqueued on the current stream after the iterator's earlier work (state), and recorded in
        state unless the caller records its own work on the chunk."""
        lib = L.lib()
        m, _keep, dev, up, B, T, mel_cl, bs, rs, lens_d, _ = inputs    # _keep: the packed weights stay alive while the stream runs
        with torch.no_grad(), torch.cuda.device(dev):
            try:
                for f0 in range(0, T, chunk_frames):
                    f1 = min(f0 + chunk_frames, T)
                    stream = state.enter()                     # after the packing and the mel's conversion, whatever their stream
                    ws = torch.empty(lib.fs2_vocoder_window_workspace_bytes(C.byref(m), B, f1 - f0), dtype=torch.uint8, device=dev)
                    n = (f1 - f0) * up
                    wav = torch.empty(B, 1, n, dtype=torch.float32, device=dev)
                    wa = L.VocoderWindowArgs(B=B, T=T, mel=mel_cl.data_ptr(), mel_batch_stride=bs, mel_row_stride=rs, wav=wav.data_ptr(),
                                             workspace=ws.data_ptr(), workspace_bytes=ws.numel(), mel_lens=L.ptr(lens_d),
                                             f0=f0, f1=f1, wav_batch_stride=n)
                    L.check(lib.fs2_vocoder_forward_window(C.byref(m), C.byref(wa), stream.cuda_stream), "fs2_vocoder_forward_window")
                    if record:
                        state.record()
                    yield f0 * up, wav
            finally:
                state.release(mel_cl, lens_d)

    def stream_pool(self, chunk_frames=64, sample_rate=None, pcm16=False, generators=()):
        """A pool of independent streams vocoded together (fs2_vocoder_forward_streams), for serving requests that arrive at different
        times: StreamPool.add(mel) admits a stream, and every StreamPool.step() synthesises the next `chunk_frames` frames of every live
        stream in one call, each at its own position.  Concatenated, one stream's chunks equal self(mel[None]) bit for bit, whatever else
        shares the pool.  It uses the weights packed at creation, like stream(); the workspace depends on the live count and
        chunk_frames, not on any length.

        sample_rate (optional): step() returns each stream's chunk at this rate, converted after the vocoder's call; a stream keeps its
        chunk count, each chunk holding the outputs whose support has arrived (the last flushes the rest), and concatenated they equal
        Resampler(h.sampling_rate, sample_rate)(self(mel[None])) bit for bit.  pcm16: int16 chunks (x 32768, truncated, clamped).
        ValueError when chunk_frames * hop is below the resampler's history.  These are the defaults of StreamPool.add, which can give
        each stream its own rate and encoding ("f32", "pcm16", "ulaw", "alaw"); every stream that is not at h.sampling_rate in fp32 is
        converted by one fs2_resample_streams_mixed launch per step, whatever its format.

        A stream whose mel arrives in pieces: h = pool.open(); pool.feed(h, block) as blocks arrive; pool.close(h) after the last.
        Its chunks, concatenated, equal self(cat(blocks)[None]) (and the conversion of that) bit for bit; its mel is held in a ring
        of StreamPool.ring_frames rows that depends on chunk_frames only, filled by one fs2_mel_ring_append launch per step.

        generators: more generators of this one's architecture (fine-tuned voices, or the reference's LJSpeech and universal
        checkpoints), vocoded in the same calls: the pool's generators are (self, *generators), and StreamPool.add / open take the
        index of a stream's generator (0, self, by default).  A stream's chunks then equal generators[k](mel[None]) bit for bit,
        whatever the other streams' generators, and a step still makes one call with the launches of a one-generator step
        (fs2_vocoder_forward_streams_multi).  Each must match self in its config (upsample_*, resblock_*, sampling_rate),
        effective_masks(), use_tensor_cores, wide_pairs and device, and be in eval mode; ValueError otherwise, and for more than
        L.MAX_GENERATORS in all.  Each is packed once, here.

        CUDA streams: every add, feed and step enqueues its device work on the stream current at that call, after the pool's earlier
        work on any other stream (its mel conversions, rings, previous chunks and generator table), with no host sync; one pool may
        be driven from several streams.  The mels the caller passes in and the chunks it gets back follow torch's usual rule: the
        caller orders them across streams.  The pool's own tensors are not freed while a stream it ran on still has queued work that
        reads them, and its workspace is allocated per step on the step's stream."""
        if isinstance(chunk_frames, bool) or not isinstance(chunk_frames, int) or chunk_frames < 1:
            raise ValueError("chunk_frames must be a positive int")
        rs = self._resampler(sample_rate, chunk_frames)
        if self.training:
            raise NotImplementedError("H100-native hifigan.Generator is inference-only: call .eval() (utils/model.py:67)")
        dev = get(self, "conv_pre.bias").device
        gens = (self, *generators)
        self._check_pool_generators(gens, dev)
        with (torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()):
            packs = [g._packed_on_stream() for g in gens]
        m, keep, dev, up = packs[0]
        lib = L.lib()
        models = L.model_array([p[0] for p in packs])
        # the generators' structs in device memory, read per work item by the multi-generator call (one upload, at its first call)
        models_dev = [None]

        def launch_multi(ptrs, f0s, ns, caps, gen):
            """One fs2_vocoder_forward_streams_multi call: stream b vocoded by generator gen[b] (its ring of caps[b] rows with caps)."""
            B, n = len(ptrs), chunk_frames * up
            with torch.cuda.device(dev):
                if models_dev[0] is None:
                    models_dev[0] = torch.frombuffer(bytearray(b"".join(bytes(p[0]) for p in packs)), dtype=torch.uint8).to(dev)
                host = torch.empty((5 if caps is None else 6) * B, dtype=torch.int32, pin_memory=True)
                h = host.numpy()
                h[:2 * B].view(np.int64)[:] = ptrs
                h[2 * B:3 * B] = f0s
                h[3 * B:4 * B] = ns
                h[4 * B:5 * B] = gen
                if caps is not None:
                    h[5 * B:] = caps
                table = host.to(dev, non_blocking=True)
                ws = torch.empty(lib.fs2_vocoder_streams_multi_workspace_bytes(models, len(packs), B, chunk_frames), dtype=torch.uint8,
                                 device=dev)
                wav = torch.empty(B, n, dtype=torch.float32, device=dev)
                base = table.data_ptr()
                a = L.VocoderStreamsMultiArgs(B=B, frames=chunk_frames, mel=base, mel_lens=base + 12 * B, f0=base + 8 * B, wav=wav.data_ptr(),
                                              wav_batch_stride=n, workspace=ws.data_ptr(), workspace_bytes=ws.numel(),
                                              cap=0 if caps is None else base + 20 * B, gen=base + 16 * B, models_dev=models_dev[0].data_ptr())
                L.check(lib.fs2_vocoder_forward_streams_multi(models, len(packs), C.byref(a), torch.cuda.current_stream(dev).cuda_stream),
                        "fs2_vocoder_forward_streams_multi")
            return wav

        def launch(ptrs, f0s, ns, caps=None, gens=None):
            """One fs2_vocoder_forward_streams call on the current stream (fs2_vocoder_forward_streams_ring with caps): uploads the
            (pointer, f0, n[, cap]) table from a fresh pinned block with one non_blocking copy (the caching host allocator keeps the
            block until the copy is done; no host sync).  gens (a pool of several generators): fs2_vocoder_forward_streams_multi."""
            if gens is not None:
                return launch_multi(ptrs, f0s, ns, caps, gens)
            B, n = len(ptrs), chunk_frames * up
            with torch.cuda.device(dev):
                host = torch.empty((4 if caps is None else 5) * B, dtype=torch.int32, pin_memory=True)
                h = host.numpy()
                h[:2 * B].view(np.int64)[:] = ptrs
                h[2 * B:3 * B] = f0s
                h[3 * B:4 * B] = ns
                if caps is not None:
                    h[4 * B:] = caps
                table = host.to(dev, non_blocking=True)
                ws = torch.empty(lib.fs2_vocoder_streams_workspace_bytes(C.byref(m), B, chunk_frames), dtype=torch.uint8, device=dev)
                wav = torch.empty(B, n, dtype=torch.float32, device=dev)
                base = table.data_ptr()
                args = dict(B=B, frames=chunk_frames, mel=base, mel_lens=base + 12 * B, f0=base + 8 * B, wav=wav.data_ptr(),
                            wav_batch_stride=n, workspace=ws.data_ptr(), workspace_bytes=ws.numel())
                st = torch.cuda.current_stream(dev).cuda_stream
                if caps is None:
                    L.check(lib.fs2_vocoder_forward_streams(C.byref(m), C.byref(L.VocoderStreamsArgs(**args)), st),
                            "fs2_vocoder_forward_streams")
                else:
                    L.check(lib.fs2_vocoder_forward_streams_ring(C.byref(m), C.byref(L.VocoderStreamsRingArgs(cap=base + 16 * B, **args)),
                                                                 st), "fs2_vocoder_forward_streams_ring")
            return wav

        def append(records):
            """One fs2_mel_ring_append launch on the current stream, its records uploaded as launch's table is."""
            with torch.cuda.device(dev):
                host = torch.empty(7 * len(records), dtype=torch.int64, pin_memory=True)
                t = host.numpy().reshape(-1, 7)
                t[:, :6] = [r[:6] for r in records]
                t[:, 6] = [r[6] | (r[7] << 32) for r in records]       # cap and count: two int32, cap first
                table = host.to(dev, non_blocking=True)
                a = L.MelRingAppendArgs(table=table.data_ptr(), n_records=len(records), n_mel=m.n_mel, max_count=max(r[7] for r in records))
                L.check(lib.fs2_mel_ring_append(C.byref(a), torch.cuda.current_stream(dev).cuda_stream), "fs2_mel_ring_append")

        def resample(records, max_out):
            with torch.cuda.device(dev):
                return Resampler.mixed(records, max_out, dev)[1]
        fs = _cfg(self.h, "sampling_rate")
        resample.rs = rs or Resampler(fs, fs)
        pool = StreamPool(launch, m.n_mel, up, chunk_frames, dev, resample=resample, encoding="pcm16" if pcm16 else "f32", append=append,
                          reach=mel_reach(m, chunk_frames), n_generators=len(gens))
        pool._keep = (packs, models, models_dev)       # the packed weights and the model tables stay alive while the pool runs
        return pool

    def _check_pool_generators(self, gens, dev):
        """ValueError unless every generator can share self's plan in one stream pool (stream_pool's generators)."""
        if len(gens) > L.MAX_GENERATORS:
            raise ValueError(f"a stream pool takes at most {L.MAX_GENERATORS} generators, got {len(gens)}")
        keys = ("upsample_rates", "upsample_kernel_sizes", "upsample_initial_channel", "resblock", "resblock_kernel_sizes",
                "resblock_dilation_sizes", "sampling_rate")
        for k, g in enumerate(gens[1:], 1):
            if not isinstance(g, Generator):
                raise ValueError(f"generators[{k}] is not a hifigan Generator")
            if g.training:
                raise ValueError(f"generators[{k}] is in training mode: call .eval()")
            if any(str(_cfg(g.h, n)) != str(_cfg(self.h, n)) for n in keys):
                raise ValueError(f"generators[{k}] has another architecture or sampling rate than generators[0]")
            if (g.effective_masks() != self.effective_masks() or bool(g.use_tensor_cores) != bool(self.use_tensor_cores)
                    or bool(g.wide_pairs) != bool(self.wide_pairs)):
                raise ValueError(f"generators[{k}]'s masks, use_tensor_cores or wide_pairs differ from generators[0]'s")
            if get(g, "conv_pre.bias").device != dev:
                raise ValueError(f"generators[{k}] is on {get(g, 'conv_pre.bias').device}, generators[0] on {dev}")


def mel_reach(m, chunk_frames):
    """(left, right): the mel frames a chunk [f0, f0 + chunk_frames) of model m reads before f0 and past f0 + chunk_frames -- conv_pre's
    input rows of the plan of a window that neither utterance end clips (L.vocoder_window_plan)."""
    f0 = 1 << 16
    pre = L.vocoder_window_plan(m, 1 << 20, f0, f0 + chunk_frames)[0]
    return f0 - pre.x0, pre.x1 - f0 - chunk_frames


class _Feed:
    """An open stream's state: the frames in its ring, the caller's blocks not yet appended ([tensor [n_mel, m], frames appended]),
    and whether it is closed."""
    __slots__ = ("written", "blocks", "closed")

    def __init__(self):
        self.written, self.blocks, self.closed = 0, collections.deque(), False


class StreamPool:
    """Streams vocoded together in chunks of `chunk_frames` mel frames (Generator.stream_pool).  Streams are kept in admission order;
    each starts at frame 0 in the step after its add() and leaves after its last chunk.  `launch(ptrs, f0s, ns)` computes one step: the
    [B, chunk_frames * up] waveform of the live streams, stream b from its frame f0s[b] of the ns[b] frames at device address ptrs[b].

    resample (optional): `resample(records, max_out)` converts one step's waveform, in one call, for every live stream whose format is
    not the waveform's own rate in fp32 (those take their slice of the waveform): records[b] = (x0, x1, i0, i1, i2, n, j0, j1,
    resampler, encoding) gives stream b's previous chunk (address x0, input samples [i0, i1)) and current chunk (x1, [i1, i2)) of its n
    samples, the outputs [j0, j1) it emits, its resample.Resampler (the identity at the waveform's rate) and its L.RESAMPLE_* encoding;
    the call returns rows indexable by b (a [B, >= max(j1 - j0)] tensor, or a list of tensors), row b starting with stream b's outputs.
    Its `.rs`, a Resampler from the waveform's rate, and `encoding` ("f32", "pcm16", "ulaw" or "alaw") are the defaults of add(); a
    pool without `resample` only vocodes.

    append (optional): what open streams (open / feed / close) need.  `append(records)` copies arriving mel frames into the streams'
    rings, in one call: records[r] = (src, frame_stride, channel_stride, src_frame, ring, dst_frame, cap, count) copies `count` frames,
    source frame src_frame + i at element src_frame + i times frame_stride, plus c times channel_stride for channel c, of the tensor at
    address src, to row (dst_frame + i) mod cap of the [cap, n_mel] ring at address ring (fs2_mel_ring_append).  reach = (left, right):
    the mel frames a chunk [f0, f0 + chunk_frames) reads before f0 and past its end (mel_reach).  In a step in which a stream opened
    with open() takes part, launch is called as launch(ptrs, f0s, ns, caps=caps): stream b's frame t at row t mod caps[b] of ptrs[b]
    (caps[b] = ns[b] for an add()ed stream, which never wraps).

    n_generators: the generators the launch call serves (Generator.stream_pool's generators).  With more than one, add() and open()
    take each stream's generator index, and launch is called with gens=[the live streams' indices] as a keyword; a one-generator
    pool calls launch(ptrs, f0s, ns[, caps]) as above."""

    def __init__(self, launch, n_mel, up, chunk_frames, device, resample=None, encoding="f32", append=None, reach=(0, 0), n_generators=1):
        self._launch, self.n_mel, self.up, self.chunk_frames, self.device = launch, n_mel, up, chunk_frames, torch.device(device)
        self._resample = resample
        rs = getattr(resample, "rs", None)
        self._rates = {} if rs is None else {rs.fs_out: rs}   # output rate -> its Resampler, one per rate
        self._default = (rs, self._encoding(encoding))
        self._append, self.reach = append, tuple(reach)
        # an open stream's ring holds the cone of its current chunk: the frames written last are at most f0 + chunk_frames + right
        self.ring_frames = -(-(self.reach[0] + chunk_frames + self.reach[1]) // 8) * 8
        self.n_generators = n_generators
        # [handle, channels-last mel view [n, n_mel] (an open stream: its ring [ring_frames, n_mel]), n (an open stream: the frames fed
        #  so far), next frame, last chunk, emitted, Resampler or None, encoding, _Feed (None for an add()ed stream), generator index]
        self._live = []
        self._next = 0
        # the pool's last enqueued work (creation: the packed weights; then every conversion, append, launch and resampling), which
        # work on another stream waits for, and the streams the pool has used, on which dropped tensors are recorded
        self._state = _streams.made(self.device)

    def _encoding(self, name):
        if name not in ENCODINGS:
            raise ValueError(f"encoding must be one of {sorted(ENCODINGS)}, got {name!r}")
        if ENCODINGS[name] != L.RESAMPLE_F32 and self._resample is None:
            raise ValueError(f"this pool has no conversion call for encoding {name!r}")
        return ENCODINGS[name]

    def _resampler(self, sample_rate):
        """The Resampler of an output rate (None: the pool's default), checked against the pool's limits."""
        if sample_rate is None:
            return self._default[0]
        default = self._default[0]
        if default is None:
            raise ValueError("this pool has no conversion call: it cannot change a stream's rate")
        rs = Resampler(default.fs_in, sample_rate)
        rs = self._rates.setdefault(rs.fs_out, rs)
        if self.chunk_frames * self.up < rs.history:
            raise ValueError(f"chunk_frames * {self.up} samples must cover the resampler's history of {rs.history} samples")
        return rs

    @staticmethod
    def _native(s):
        """The stream takes its slice of the waveform: its rate is the waveform's and its encoding fp32."""
        return (s[6] is None or s[6].identity) and s[7] == L.RESAMPLE_F32

    def _generator(self, generator):
        """A new stream's generator index, checked against the pool's generators."""
        if isinstance(generator, bool) or not isinstance(generator, int) or not 0 <= generator < self.n_generators:
            raise ValueError(f"generator must be an int in [0, {self.n_generators}), got {generator!r}")
        return generator

    def add(self, mel, sample_rate=None, encoding=None, generator=0):
        """Admits a stream.  mel: [n_mel, n] or [1, n_mel, n] on the pool's device, n >= 1.  A channels-last view with row stride n_mel
        (FastSpeech2's postnet_mel[b, :n].T is one) is kept without a copy; any other layout is converted once.  sample_rate and encoding
        ("f32", "pcm16", "ulaw" or "alaw"): the stream's output format, None for the pool's.  ValueError for a rate Resampler refuses, a
        resampler history longer than chunk_frames * up, an unknown encoding, or a ninth distinct output rate among the live streams.
        generator: the index of the stream's generator in the pool's (ValueError outside them).  Returns the handle."""
        generator = self._generator(generator)
        if not isinstance(mel, torch.Tensor):
            raise ValueError("mel must be a tensor")
        if mel.dim() == 3 and mel.shape[0] == 1:
            mel = mel[0]
        if mel.dim() != 2 or mel.shape[0] != self.n_mel:
            raise ValueError(f"expected mel of shape [{self.n_mel}, n] or [1, {self.n_mel}, n]")
        if mel.device != self.device:
            raise ValueError(f"mel is on {mel.device}, the vocoder on {self.device}")
        n = mel.shape[1]
        if n < 1:
            raise ValueError("mel has no frames")
        rs, enc = self._format(sample_rate, encoding)
        rows = mel.T
        if not (rows.dtype == torch.float32 and rows.stride(1) == 1 and (n == 1 or rows.stride(0) == self.n_mel) and rows.data_ptr() % 16 == 0):
            self._state.enter()
            rows = rows.to(torch.float32).contiguous()
            self._state.record()
        return self._admit(rows, n, rs, enc, None, generator)

    def _format(self, sample_rate, encoding):
        """A new stream's (Resampler or None, encoding), checked as add() documents."""
        rs = self._resampler(sample_rate)
        enc = self._default[1] if encoding is None else self._encoding(encoding)
        rates = {s[6].fs_out for s in self._live if s[6] is not None}
        if rs is not None and rs.fs_out not in rates and len(rates) >= L.RESAMPLE_MAX_FILTERS:
            raise ValueError(f"the live streams already use {len(rates)} output rates; at most {L.RESAMPLE_MAX_FILTERS}")
        return rs, enc

    def _admit(self, rows, n, rs, enc, feed, generator):
        h = self._next
        self._next += 1
        self._live.append([h, rows, n, 0, None, 0, rs, enc, feed, generator])
        return h

    def open(self, sample_rate=None, encoding=None, generator=0):
        """Admits a stream whose mel has not arrived yet: feed(h, block) appends frames, close(h) fixes its length.  It takes part in a
        step once its next chunk's cone has arrived, and concatenated its chunks equal those of add() on the concatenated blocks bit
        for bit.  Its mel lives in a ring of ring_frames rows, whatever its length.  sample_rate, encoding and generator as in add().
        ValueError in a pool without an append call.  Returns the handle."""
        generator = self._generator(generator)
        if self._append is None:
            raise ValueError("this pool has no append call: it cannot take open streams")
        rs, enc = self._format(sample_rate, encoding)
        ring = torch.empty(self.ring_frames, self.n_mel, dtype=torch.float32, device=self.device)
        return self._admit(ring, 0, rs, enc, _Feed(), generator)

    def _open_stream(self, h):
        for s in self._live:
            if s[0] == h:
                if s[8] is None:
                    raise ValueError(f"stream {h} was admitted whole by add()")
                if s[8].closed:
                    raise ValueError(f"stream {h} is closed")
                return s
        raise KeyError(h)

    def feed(self, h, mel):
        """Queues the next frames of open stream h: mel [n_mel, m] or [1, n_mel, m], m >= 1, on the pool's device, in any layout
        (FastSpeech2's postnet_mel[b, a:z].T and a channel-major [n_mel, m] block are both read in place).  The pool keeps a reference
        to the tensor until its last frame has been copied into the ring; the caller must not write it before then.  A floating
        block that is not fp32 is converted once.  KeyError for a handle that is not live, ValueError for a closed or add()ed stream
        or a bad block."""
        s = self._open_stream(h)
        if not isinstance(mel, torch.Tensor):
            raise ValueError("mel must be a tensor")
        if mel.dim() == 3 and mel.shape[0] == 1:
            mel = mel[0]
        if mel.dim() != 2 or mel.shape[0] != self.n_mel:
            raise ValueError(f"expected mel of shape [{self.n_mel}, m] or [1, {self.n_mel}, m]")
        if mel.device != self.device:
            raise ValueError(f"mel is on {mel.device}, the vocoder on {self.device}")
        if not mel.dtype.is_floating_point:
            raise ValueError(f"mel must be floating point, got {mel.dtype}")
        if mel.shape[1] < 1:
            raise ValueError("mel has no frames")
        if mel.dtype != torch.float32:
            self._state.enter()
            mel = mel.to(torch.float32)
            self._state.record()
        s[8].blocks.append([mel, 0])
        s[2] += mel.shape[1]

    def close(self, h):
        """Fixes open stream h's length at the frames fed so far; its remaining chunks then take part in every step, the last trimmed
        to its end.  A stream closed with no frames leaves without output.  KeyError / ValueError as feed()."""
        s = self._open_stream(h)
        s[8].closed = True
        if s[3] >= s[2]:
            self._live = [x for x in self._live if x is not s]
            self._drop(s)

    def cancel(self, h):
        """Drops a live stream (KeyError if it is not live)."""
        for i, s in enumerate(self._live):
            if s[0] == h:
                del self._live[i]
                self._drop(s)
                return
        raise KeyError(h)

    def _drop(self, s):
        """Releases the device tensors of stream record s, which has left the pool."""
        self._state.release(s[1], s[4], *(b[0] for b in (s[8].blocks if s[8] is not None else ())))

    def __len__(self):
        return len(self._live)

    def step(self):
        """One chunk of every live stream, in one launch call: a list of (handle, first_sample, chunk [1, 1, m]) in admission order,
        m = chunk_frames * up except on a stream's last chunk, which is trimmed to its end.  [] without a call when the pool is empty.
        A converted stream: first_sample and m at its own rate, the chunk holding the outputs that became ready (possibly none), of its
        encoding's dtype; at most one conversion call per step, none when every live stream is at the waveform's rate in fp32.

        An open stream takes part only once the cone of its next chunk has arrived (fed >= f0 + chunk_frames + reach[1]), or once it is
        closed; a starved one yields nothing and holds nobody back, and a step in which no stream takes part makes no call.  In a step
        with a stream from open(), one append call first copies into the rings the frames this step's chunks read, then the launch
        runs every stream that takes part on rings (launch's caps)."""
        live = [s for s in self._live if s[8] is None or s[8].closed or s[2] >= s[3] + self.chunk_frames + self.reach[1]]
        if not live:
            return []
        self._state.enter()
        ptrs, f0s, ns = [s[1].data_ptr() for s in live], [s[3] for s in live], [s[2] for s in live]
        gens = {} if self.n_generators == 1 else {"gens": [s[9] for s in live]}
        if any(s[8] is not None for s in live):
            self._fill(live)
            wav = self._launch(ptrs, f0s, ns, caps=[n if s[8] is None else self.ring_frames for s, n in zip(live, ns)], **gens)
        else:
            wav = self._launch(ptrs, f0s, ns, **gens)
        rows = [(wav, i) for i in range(len(live))]     # where each stream's chunk is: (rows, index)
        starts = [s[3] * self.up for s in live]
        widths = [min(self.chunk_frames, s[2] - s[3]) * self.up for s in live]
        conv = [i for i, s in enumerate(live) if not self._native(s)]
        if conv:
            y = self._converted(live, conv, wav, starts, widths)
            for k, i in enumerate(conv):
                rows[i] = (y, k)
        out = []
        for i, s in enumerate(live):
            t, k = rows[i]
            out.append((s[0], starts[i], t[k][None, None, :widths[i]]))
            s[3] += self.chunk_frames
        self._state.record()
        keep = [s for s in self._live if (s[8] is not None and not s[8].closed) or s[3] < s[2]]
        for s in live:
            if (s[8] is None or s[8].closed) and s[3] >= s[2]:
                self._drop(s)
        self._live = keep
        return out

    def _fill(self, live):
        """One append call copying, for each stream from open() among `live`, its frames up to the end of this step's cone (or its
        end) that are not in its ring yet."""
        records, done = [], []
        for s in live:
            f = s[8]
            if f is None:
                continue
            target = min(s[3] + self.chunk_frames + self.reach[1], s[2])
            while f.written < target:
                blk = f.blocks[0]
                mel, off = blk
                k = min(mel.shape[1] - off, target - f.written)
                records.append((mel.data_ptr(), mel.stride(1), mel.stride(0), off, s[1].data_ptr(), f.written, self.ring_frames, k))
                f.written += k
                blk[1] = off + k
                if blk[1] == mel.shape[1]:
                    done.append(f.blocks.popleft())
        if records:
            self._append(records)
        # The blocks appended in full are released only now, after the call is enqueued (the rule _converted states for its chunks).
        self._state.release(*(b[0] for b in done))
        del done

    def _converted(self, live, conv, wav, starts, widths):
        """The conversion call for streams `conv` on this step's waveform; sets their first output and output count in starts and
        widths."""
        n1 = self.chunk_frames * self.up
        records = []
        for i in conv:
            s = live[i]
            _, _, n, f0, prev, emitted, rs, enc, feed, _ = s
            i1, N = f0 * self.up, n * self.up              # an open stream: N covers every input its ready outputs read
            is_open = feed is not None and not feed.closed
            r = rs.ready(min(i1 + n1, N), None if is_open else N, not is_open and f0 + self.chunk_frames >= n)
            cur = wav[i]
            records.append((0 if prev is None else prev.data_ptr(), cur.data_ptr(), i1 - (0 if prev is None else n1), i1, i1 + n1, N,
                            emitted, r, rs, enc))
            starts[i], widths[i] = emitted, r - emitted
            s[5] = r
        y = self._resample(records, max(widths[i] for i in conv))
        # Each chunk stays alive as the next step's history.  The previous chunks are released only now: the call is enqueued, so a
        # later allocation that reuses their memory is written after the call has read them (released before, the call's own table
        # upload or output could take that memory first).
        self._state.release(*(live[i][4] for i in conv))
        for i in conv:
            live[i][4] = wav[i]
        return y
