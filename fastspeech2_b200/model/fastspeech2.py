"""Drop-in `model.fastspeech2.FastSpeech2`: same constructor, state_dict keys, forward signature and 10-tuple as the
reference (model/fastspeech2.py:13-110); the forward itself is hand-written sm_90a CUDA behind the C ABI
(include/fs2b200.h: fs2_acoustic_encode + fs2_acoustic_decode).  Inference only; there is no PyTorch fallback.
"""
from __future__ import annotations

import contextlib
import ctypes as C

import torch
import torch.nn as nn

from .. import _lib as L
from .. import _streams
from .. import packing
from .._modtree import get, populate
from ..spec import fastspeech2_spec, read_dataset_files
from ..synth import sinusoid_table

_UNREAD_CONTROL = (None, 1.0, (0, 0))


def normalize_control(control, shape, device, name="control"):
    """A p_control / d_control argument as the C ABI takes it (fs2_control_args), for the prediction of `shape` ([B, L] phonemes or
    [B, T] frames) that it scales as the reference's `prediction * control` does (model/modules.py:85,96,134).  Returns
    (tensor, scalar, strides):
      * a Python number or a one-element tensor: (None, float(control), (0, 0)), the scalar path;
      * any other tensor: (an fp32 view on `device` broadcast to `shape`, 1.0, its two element strides).  Dimensions the tensor
        broadcasts along (size 1, or stride 0 in an expanded view) get stride 0: the values are converted, never materialised.
    Raises ValueError for a tensor that does not broadcast to `shape` (the reference raises too) or that would grow it, e.g.
    [B, L, 1] (torch.broadcast_shapes(control.shape, shape) != shape; the reference would silently grow every later tensor)."""
    if not torch.is_tensor(control) or control.numel() == 1:
        return None, float(control), (0, 0)
    shape = torch.Size(shape)
    if control.is_complex():
        raise ValueError(f"{name} must be real, got {control.dtype}")
    try:
        full = torch.broadcast_shapes(control.shape, shape)
    except RuntimeError as e:
        raise ValueError(f"{name} of shape {tuple(control.shape)} does not broadcast to the prediction's shape {tuple(shape)}") from e
    if full != shape:
        raise ValueError(f"{name} of shape {tuple(control.shape)} would grow the prediction's shape {tuple(shape)} to {tuple(full)}")
    compact = control[tuple(slice(0, 1) if st == 0 else slice(None) for st in control.stride())]
    view = compact.to(device=device, dtype=torch.float32).broadcast_to(shape)
    return view, 1.0, tuple(view.stride())


def _control_args(p, d):
    c = L.ControlArgs()
    if p[0] is not None:
        c.p, (c.p_stride_b, c.p_stride_l) = p[0].data_ptr(), p[2]
    if d[0] is not None:
        c.d, (c.d_stride_b, c.d_stride_l) = d[0].data_ptr(), d[2]
    return c


class FastSpeech2(nn.Module):
    """FastSpeech2 acoustic model, H100-native forward.

    Arguments, parameter names and return values mirror the reference class (model/fastspeech2.py:16-41,:43-110).
    """

    # Ragged mode, per instance or for the class (forward's `ragged` overrides it per call): utterance b is synthesised from its own
    # src_lens[b] phonemes and mel_lens[b] frames only, bit for bit as it would be alone, and the padding's work is skipped
    # (fs2_acoustic_encode_ragged in fs2b200.h).  Off: the reference's batched semantics, in which padded rows reach the last phonemes
    # and frames of every shorter utterance.
    ragged = False

    def __init__(self, preprocess_config, model_config):
        super().__init__()
        self.model_config = model_config
        self.preprocess_config = preprocess_config
        pp = preprocess_config["preprocessing"]
        self.pitch_feature_level = pp["pitch"]["feature"]
        self.energy_feature_level = pp["energy"]["feature"]
        for lvl in (self.pitch_feature_level, self.energy_feature_level):
            assert lvl in ("phoneme_level", "frame_level")
        ve = model_config["variance_embedding"]
        for q in (ve["pitch_quantization"], ve["energy_quantization"]):
            assert q in ("linear", "log")
        stats, _ = read_dataset_files(preprocess_config)
        self._spec = fastspeech2_spec(preprocess_config, model_config)
        populate(self, self._spec, stats)
        if ve["pitch_quantization"] == "log" or ve["energy_quantization"] == "log":
            import numpy as np  # log-spaced edges, model/modules.py:48-54,:60-67
            n = ve["n_bins"] - 1
            with torch.no_grad():
                if ve["pitch_quantization"] == "log":
                    get(self, "variance_adaptor.pitch_bins").copy_(
                        torch.exp(torch.linspace(np.log(stats["pitch"][0]), np.log(stats["pitch"][1]), n)))
                if ve["energy_quantization"] == "log":
                    get(self, "variance_adaptor.energy_bins").copy_(
                        torch.exp(torch.linspace(np.log(stats["energy"][0]), np.log(stats["energy"][1]), n)))
        self.multi_speaker = bool(model_config["multi_speaker"])
        self.max_seq_len = int(model_config["max_seq_len"])
        # Which sub-networks run on the tensor-core kernels (L.TC_* bits; cleared = exact fp32 CUDA-core kernels).
        #  * decoder FFT blocks, mel_linear, PostNet: two-MMA operand split (*_F8: fp16 main term + one E4M3 correction MMA), fused attention.
        #  * encoder FFT blocks and the three variance predictors feed the DISCRETE duration / pitch / energy-bucket decisions (SURVEY.md
        #    section 7, hard part 2).  A single long tensor-core accumulation (432 truncating steps for the k = 9 conv) flips buckets
        #    noticeably more often than the fp32 kernels.  They therefore run K-SEGMENTED (fs2b200.h: every (tap, 256-channel) slice is
        #    its own 16-step work unit with a separate hi*hi accumulator, slices summed in fp32 round-to-nearest), which brings the flips
        #    back to the fp32 kernels' level (scripts/flip_census.py).  Clear the two bits for the fp32 kernels.
        self.tc_mask = (L.TC_DECODER | L.TC_POSTNET | L.TC_DECODER_F8 | L.TC_POSTNET_F8 | L.TC_ENCODER | L.TC_PREDICTORS)
        self._packed = None          # (AcousticModel struct, keep-alive tensors, device)
        self._packed_state = None    # _streams.StreamState of the packed weights: made on the stream of the call that packed them
        self._pos_long = {}          # width -> (device position table longer than max_seq_len, its StreamState)
        self._ws, self._ws_stream = None, None     # the last call's workspace and the stream it was allocated on (_streams.workspace)
        self._stats_host = None      # the last call's len_stats [max, sum of mel_lens, wild durations], pinned, final once its stream syncs

    # ------------------------------------------------------------------ packing
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

    def repack(self):
        """Call after mutating parameters in place."""
        self._invalidate()

    def _pack(self):
        L.lib()
        tr = self.model_config["transformer"]
        vp = self.model_config["variance_predictor"]
        if tr["encoder_hidden"] != tr["decoder_hidden"] or tr["encoder_head"] != tr["decoder_head"]:
            raise L.Fs2Error("encoder/decoder width or head count differ: unsupported by the sm_90a kernels")
        dev = get(self, "mel_linear.weight").device
        if dev.type != "cuda":
            raise L.Fs2Error("FastSpeech2 (H100-native) needs its parameters on a CUDA device; there is no CPU path")
        n_post = 0
        while f"postnet.convolutions.{n_post}.0.conv.weight" in self._keys():
            n_post += 1
        pk = packing.pack_acoustic(lambda k: get(self, k).detach().float(), tr["encoder_layer"], tr["decoder_layer"], n_post,
                                   self.multi_speaker, f8_decoder=bool(self.tc_mask & L.TC_DECODER_F8),
                                   f8_postnet=bool(self.tc_mask & L.TC_POSTNET_F8))
        m = L.AcousticModel()
        m.d_model, m.n_head, m.d_inner = tr["encoder_hidden"], tr["encoder_head"], tr["conv_filter_size"]
        m.k1, m.k2 = tr["conv_kernel_size"]
        m.n_enc, m.n_dec = tr["encoder_layer"], tr["decoder_layer"]
        m.n_mel = self.preprocess_config["preprocessing"]["mel"]["n_mel_channels"]
        m.vp_filter, m.vp_kernel = vp["filter_size"], vp["kernel_size"]
        m.n_bins = self.model_config["variance_embedding"]["n_bins"]
        m.n_vocab = pk["word_emb"].shape[0]
        if m.n_enc > L.MAX_LAYERS or m.n_dec > L.MAX_LAYERS or n_post > L.MAX_POSTNET:
            raise L.Fs2Error("model exceeds the C ABI's fixed table sizes")
        P = lambda k: pk[k].data_ptr()
        m.word_emb, m.enc_pos, m.dec_pos = P("word_emb"), P("enc_pos"), P("dec_pos")
        m.enc_pos_rows = m.dec_pos_rows = self.max_seq_len + 1
        self._pos_ptrs = (m.enc_pos, m.dec_pos)
        m.spk_emb, m.n_speakers = (P("spk_emb"), pk["spk_emb"].shape[0]) if self.multi_speaker else (0, 0)
        for side, n in (("enc", m.n_enc), ("dec", m.n_dec)):
            for i in range(n):
                dst = getattr(m, side)[i]
                for name, _ in L.FftBlockWeights._fields_:
                    key = f"{side}.{i}.{name}"
                    setattr(dst, name, P(key) if key in pk else 0)
        for nm in ("dur", "pitch", "energy"):
            dst = getattr(m, nm)
            for name, _ in L.PredictorWeights._fields_:
                key = f"{nm}.{name}"
                setattr(dst, name, P(key) if key in pk else 0)
        for name in ("pitch_bins", "energy_bins", "pitch_emb", "energy_emb", "w_mel", "b_mel"):
            setattr(m, name, P(name))
        m.tc_mask = self.tc_mask
        m.pitch_frame_level = int(self.pitch_feature_level == "frame_level")
        m.energy_frame_level = int(self.energy_feature_level == "frame_level")
        m.w_mel_tc = P("w_mel_tc") if "w_mel_tc" in pk else 0
        m.n_postnet = n_post
        for i in range(n_post):
            m.w_post_tc[i] = P(f"post.{i}.w_tc") if f"post.{i}.w_tc" in pk else 0
            w = pk[f"post.{i}.w"]                      # [k][cin][cout]
            m.w_post[i], m.b_post[i] = w.data_ptr(), P(f"post.{i}.b")
            m.post_k, m.post_cin[i], m.post_cout[i] = w.shape[0], w.shape[1], w.shape[2]
        self._packed = (m, pk, dev)
        self._packed_state = _streams.made(dev)
        return self._packed

    def _keys(self):
        if not hasattr(self, "_keyset"):
            self._keyset = {p.key for p in self._spec}
        return self._keyset

    def _position(self, which: int, n: int, width: int, dev):
        """Device position table with >= n rows.  Up to max_seq_len the cached parameter is used; beyond it the eval-mode
        reference recomputes the table on the fly (transformer/Models.py:82-87,:145-152) -- same here, cached by size."""
        if n <= self.max_seq_len:
            return self._pos_ptrs[which], self.max_seq_len + 1
        old = self._pos_long.get(width)
        if old is None or old[0].shape[0] < n or old[0].device != dev:
            if old is not None:
                old[1].release(old[0])
            rows = max(2048, 1 << (n - 1).bit_length())
            tab = sinusoid_table(rows, width).to(dev)
            self._pos_long[width] = (tab, _streams.made(dev))      # the upload is ordered on the current stream only
        tab, state = self._pos_long[width]
        state.enter()
        return tab.data_ptr(), tab.shape[0]

    def _workspace(self, nbytes: int, dev):
        self._ws, self._ws_stream = _streams.workspace((self._ws, self._ws_stream), nbytes, dev, grow=1.25, slack=1024)
        return self._ws

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, speakers, texts, src_lens, max_src_len, mels=None, mel_lens=None, max_mel_len=None,
                p_targets=None, e_targets=None, d_targets=None, p_control=1.0, e_control=1.0, d_control=1.0, ragged=None):
        """The reference's forward; `ragged` (None: the module's `ragged` attribute) selects the ragged mode described in __init__.

        Controls, as the reference applies them (model/modules.py:85,96,132-135): a Python number, or a tensor of any real dtype on any
        device that broadcasts, under torch rules, to the prediction it scales -- p_control to the pitch AND energy predictions
        ([B, L]; [B, T] for frame-level predictors), d_control to the durations ([B, L]).  So [B, 1] is one value per utterance and
        [B, L] one per phoneme.  A 1-D control of length n is per COLUMN, exactly as in the reference: [B] is not per utterance (it
        raises unless B == L, and then scales phonemes).  A control that does not broadcast, or that would grow the prediction (e.g.
        [B, L, 1]), raises ValueError before the phase that uses it is launched.  Controls the reference never reads are accepted
        whatever they are: e_control always (model/modules.py:124), p_control when every predictor it scales is given its target,
        d_control with d_targets.  Tensor values are rounded to fp32 on the model's device without a host synchronisation; the one
        deviation from the reference is a float64 control, which the reference would let promote the prediction to float64.  Ragged
        mode: utterance b equals its solo call with c[b] ([B, 1]) or c[b:b+1, :src_lens[b]] ([B, L]), and control columns beyond an
        utterance's length are never read.

        CUDA streams: the call enqueues all of its device work on the stream current at the call; without max_mel_len it synchronises
        that stream once, to read the output length.  Its workspace is cached for the next call on the same stream only: a call on
        another stream allocates its own, so calls on two streams never share one.  The arguments and the returned tensors follow
        torch's usual rule: the caller orders them across streams.  The weights packed by the first call and the position tables
        longer than max_seq_len are ready on whatever stream a later call uses, and are not freed while another stream's queued work
        reads them."""
        # the C ABI sets up per-device kernel attributes for the CURRENT device: make the model's device current
        dev = get(self, "mel_linear.weight").device
        with (torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()):
            return self._forward(speakers, texts, src_lens, max_src_len, mels, mel_lens, max_mel_len, p_targets, e_targets, d_targets,
                                 p_control, e_control, d_control, self.ragged if ragged is None else bool(ragged))

    def _forward(self, speakers, texts, src_lens, max_src_len, mels=None, mel_lens=None, max_mel_len=None,
                 p_targets=None, e_targets=None, d_targets=None, p_control=1.0, e_control=1.0, d_control=1.0, ragged=False, voices=None):
        """forward, or with voices = (bank, voice) the VoiceBank call whose voice 0 is self."""
        for mk in (self,) if voices is None else voices[0].models:
            if mk.training:
                raise NotImplementedError("H100-native FastSpeech2 is inference-only: call .eval() (utils/model.py:32)")
        p_frame = self.pitch_feature_level == "frame_level"
        e_frame = self.energy_feature_level == "frame_level"
        L.lib()
        if voices is not None:                         # checked before any packing or device work
            voices = (voices[0], voices[0]._voice_table(voices[1], int(texts.shape[0]), get(self, "mel_linear.weight").device))
        for mk in (self,) if voices is None else voices[0].models:
            mk._packed or mk._pack()
            mk._packed_state.enter()
        m, _keep, dev = self._packed
        B, Lmax = int(texts.shape[0]), int(max_src_len)
        if texts.shape[1] != Lmax:
            raise ValueError("texts.shape[1] must equal max_src_len")
        if d_targets is not None and mel_lens is None:
            raise ValueError("d_targets needs mel_lens/max_mel_len (the reference derives the decoder mask from them)")
        i64 = dict(dtype=torch.long, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        texts = texts.to(**i64).contiguous()
        src_lens_in = src_lens
        src_lens32 = src_lens.to(device=dev, dtype=torch.int32).contiguous()
        speakers_d = speakers.to(**i64).contiguous() if (self.multi_speaker and speakers is not None) else None
        stream = torch.cuda.current_stream(dev).cuda_stream

        p_pred = torch.empty(B, Lmax, **f32); e_pred = torch.empty(B, Lmax, **f32)
        logd = torch.empty(B, Lmax, **f32); d_rounded = torch.empty(B, Lmax, **f32)
        mel_lens_out = torch.empty(B, **i64)
        mel_lens32 = torch.empty(B, dtype=torch.int32, device=dev)
        cum = torch.empty(B, Lmax, dtype=torch.int32, device=dev)
        x_adapted = torch.empty(B, Lmax, m.d_model, **f32)
        stats_dev = torch.empty(3, dtype=torch.int32, device=dev)
        # a pinned block of this call's own, filled by a torch copy on the call's stream: the caching host allocator then keeps the block
        # from reuse until that copy is done, whenever the block is dropped
        stats_host = torch.empty(3, dtype=torch.int32, pin_memory=True)
        tgt = lambda t: None if t is None else t.to(**f32).contiguous()
        p_t, e_t, d_t = tgt(p_targets), tgt(e_targets), tgt(d_targets)
        # p_control scales the predictors without a target; e_control is never read (model/modules.py:124)
        p_read_enc = (not p_frame and p_t is None) or (not e_frame and e_t is None)
        p_read_dec = (p_frame and p_t is None) or (e_frame and e_t is None)
        p_enc = normalize_control(p_control, (B, Lmax), dev, "p_control") if p_read_enc else _UNREAD_CONTROL
        d_ctl = normalize_control(d_control, (B, Lmax), dev, "d_control") if d_t is None else _UNREAD_CONTROL

        ea = L.EncodeArgs(B=B, L=Lmax, texts=texts.data_ptr(), speakers=L.ptr(speakers_d), src_lens=src_lens32.data_ptr(),
                          p_control=p_enc[1], e_control=1.0, d_control=d_ctl[1],
                          p_target=0 if p_frame else L.ptr(p_t), e_target=0 if e_frame else L.ptr(e_t), d_target=L.ptr(d_t),
                          p_pred=0 if p_frame else p_pred.data_ptr(), e_pred=0 if e_frame else e_pred.data_ptr(), logd_pred=logd.data_ptr(),
                          d_rounded=d_rounded.data_ptr(), mel_lens=mel_lens_out.data_ptr(), mel_lens32=mel_lens32.data_ptr(),
                          cum_dur=cum.data_ptr(), x_adapted=x_adapted.data_ptr(), len_stats=stats_dev.data_ptr(),
                          len_stats_host=0)
        self._phase("encode", B, Lmax, ea, _control_args(p_enc, d_ctl), ragged, stream, dev, voices)
        stats_host.copy_(stats_dev, non_blocking=True)
        self._stats_host = stats_host

        if max_mel_len is not None:
            T = int(max_mel_len)
        else:
            # the one unavoidable host sync: the output shape depends on the predicted durations (utils/tools.py:94)
            torch.cuda.current_stream(dev).synchronize()
            T = int(stats_host[0])
            if int(stats_host[2]) != 0:
                raise L.Fs2Error(f"{int(stats_host[2])} predicted durations are NaN / inf / > 1e6 frames "
                                 "(the reference raises on them too, model/modules.py:186)")
        if T <= 0:
            raise L.Fs2Error("all predicted durations are zero: nothing to decode")
        if mel_lens is not None and d_targets is not None:
            mask_lens32 = mel_lens.to(device=dev, dtype=torch.int32).contiguous()   # teacher forcing: the caller's mask (fastspeech2.py:60-64)
        else:
            mask_lens32 = mel_lens32       # free-running: the adaptor rebuilds the mask from the predicted lengths (modules.py:132-137)

        mel = torch.empty(B, T, m.n_mel, **f32)
        post = torch.empty(B, T, m.n_mel, **f32)
        if p_frame:                                    # frame-level predictions have the mel time axis (model/modules.py:139-148)
            p_pred = torch.empty(B, T, **f32)
            if p_t is not None and tuple(p_t.shape) != (B, T):
                raise ValueError("frame-level p_targets must be [B, max_mel_len]")
        if e_frame:
            e_pred = torch.empty(B, T, **f32)
            if e_t is not None and tuple(e_t.shape) != (B, T):
                raise ValueError("frame-level e_targets must be [B, max_mel_len]")
        p_dec = normalize_control(p_control, (B, T), dev, "p_control") if p_read_dec else _UNREAD_CONTROL
        da = L.DecodeArgs(B=B, L=Lmax, T=T, x_adapted=x_adapted.data_ptr(), cum_dur=cum.data_ptr(),
                          mel_mask_lens=mask_lens32.data_ptr(), p_control=p_dec[1],
                          p_target_frames=L.ptr(p_t) if p_frame else 0, e_target_frames=L.ptr(e_t) if e_frame else 0,
                          p_pred_frames=p_pred.data_ptr() if p_frame else 0, e_pred_frames=e_pred.data_ptr() if e_frame else 0,
                          mel=mel.data_ptr(), postnet_mel=post.data_ptr())
        self._phase("decode", B, T, da, _control_args(p_dec, _UNREAD_CONTROL), ragged, stream, dev, voices)

        src_masks = torch.arange(Lmax, device=dev)[None, :] >= src_lens32[:, None]
        mel_masks = torch.arange(T, device=dev)[None, :] >= mask_lens32[:, None]
        return (mel, post, p_pred, e_pred, logd, d_targets if d_targets is not None else d_rounded,
                src_masks, mel_masks, src_lens_in, mel_lens_out)

    def _phase(self, kind, B, n, args, ctl, ragged, stream, dev, voices):
        """Phase `kind` of the call ("encode": n = L phonemes, "decode": n = T frames) on self, or with voices = (bank, device voice
        table) on the bank's voices: each model's position table of >= n rows, the workspace, the call."""
        lib = L.lib()
        enc = kind == "encode"
        for mk in (self,) if voices is None else voices[0].models:
            m = mk._packed[0]
            if enc:
                m.enc_pos, m.enc_pos_rows = mk._position(0, n, m.d_model, dev)
            else:
                m.dec_pos, m.dec_pos_rows = mk._position(1, n, m.d_model, dev)
        if voices is None:
            target, owner, keep = C.byref(self._packed[0]), self, None
            size, run = getattr(lib, f"fs2_{kind}_workspace_bytes"), getattr(lib, f"fs2_acoustic_{kind}_ctl")
        else:
            owner = voices[0]
            va, keep = owner._upload(voices[1], dev)
            target = C.byref(va)
            size, run = getattr(lib, f"fs2_{kind}_voices_workspace_bytes"), getattr(lib, f"fs2_acoustic_{kind}_voices")
        ws = owner._workspace(size(target, B, n), dev)
        args.workspace, args.workspace_bytes = ws.data_ptr(), ws.numel()
        L.check(run(target, C.byref(args), C.byref(ctl), int(ragged), stream), f"fs2_acoustic_{kind}")
        del keep


def _layout(model):
    """What shapes a FastSpeech2's packed struct: its state's keys and shapes and the variance feature levels"""
    return (model.pitch_feature_level, model.energy_feature_level, tuple((k, tuple(v.shape)) for k, v in model.state_dict().items()))


class VoiceBank:
    """Several FastSpeech2 voices of one config in one acoustic call: utterance b of a batch is synthesised by models[voice[b]].

    models: 1 to L.MAX_VOICES FastSpeech2 modules of one config (the same state keys and shapes, feature levels and tc_mask), on one
    device and in eval mode, such as one fine-tuned checkpoint per voice; voice 0 is models[0].  Each voice keeps its own weights and
    tables: word and speaker embeddings, pitch / energy bins (from its own stats.json) and embeddings, and position tables.

    bank(voice, speakers, texts, src_lens, max_src_len, ...) takes FastSpeech2.forward's arguments after `voice`, an integer tensor [B]
    on any device, and returns forward's 10-tuple:
      * ragged: utterance b equals models[voice[b]] called alone on its slice with ragged=True, bit for bit;
      * padded: with T the call's output length, row b of every output equals row b of models[voice[b]] called on the same batch with
        max_mel_len=T (no kernel mixes batch rows, only where the weights come from changes).
    The call makes the launches of models[0].forward at the same B, L and T, whatever the voice mix, and never reads a device `voice`
    on the host: an index outside [0, len(models)) there gives that utterance mel_lens 0 and zero durations, leaves the others
    unchanged, and leaves its other outputs unspecified.  A CPU `voice` is checked: an index out of range raises ValueError.
    CUDA streams as in forward: the call enqueues on the current stream, synchronises it once without max_mel_len, and caches its
    workspace per stream; every voice's packed weights are ready on the calling stream."""

    def __init__(self, models):
        models = tuple(models)
        if not 1 <= len(models) <= L.MAX_VOICES:
            raise ValueError(f"a VoiceBank takes 1 to {L.MAX_VOICES} FastSpeech2 models, got {len(models)}")
        m0 = models[0]
        for k, mk in enumerate(models):
            if not isinstance(mk, FastSpeech2):
                raise ValueError(f"models[{k}] is not a FastSpeech2")
            if mk.training:
                raise ValueError(f"models[{k}] is in training mode: call .eval()")
            if _layout(mk) != _layout(m0):
                raise ValueError(f"models[{k}]'s config (state shapes or feature levels) differs from models[0]'s")
            if mk.tc_mask != m0.tc_mask:
                raise ValueError(f"models[{k}].tc_mask differs from models[0]'s")
            if get(mk, "mel_linear.weight").device != get(m0, "mel_linear.weight").device:
                raise ValueError(f"models[{k}] is on {get(mk, 'mel_linear.weight').device}, models[0] on {get(m0, 'mel_linear.weight').device}")
        self.models = models
        self._ws, self._ws_stream = None, None     # as FastSpeech2's: the last call's workspace and its stream

    def __call__(self, voice, speakers, texts, src_lens, max_src_len, mels=None, mel_lens=None, max_mel_len=None,
                 p_targets=None, e_targets=None, d_targets=None, p_control=1.0, e_control=1.0, d_control=1.0, ragged=None):
        m0 = self.models[0]
        dev = get(m0, "mel_linear.weight").device
        with (torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()):
            return m0._forward(speakers, texts, src_lens, max_src_len, mels, mel_lens, max_mel_len, p_targets, e_targets, d_targets,
                               p_control, e_control, d_control, m0.ragged if ragged is None else bool(ragged), voices=(self, voice))

    def _voice_table(self, voice, B, dev):
        """`voice` as the int32 device table the C ABI reads; ValueError for a wrong shape or dtype, or a CPU index out of range."""
        if not torch.is_tensor(voice) or voice.dtype == torch.bool or voice.is_floating_point() or voice.is_complex():
            raise ValueError(f"voice must be an integer tensor, got {voice.dtype if torch.is_tensor(voice) else type(voice).__name__}")
        if tuple(voice.shape) != (B,):
            raise ValueError(f"voice must have shape [{B}] (one voice per utterance), got {tuple(voice.shape)}")
        n = len(self.models)
        if voice.device.type == "cpu" and B and not (0 <= int(voice.min()) and int(voice.max()) < n):
            raise ValueError(f"voice indices must lie in [0, {n}), got {voice.tolist()}")
        if voice.dtype != torch.int32:
            voice = voice.clamp(-1, n)                 # a wide index stays out of range in int32
        return voice.to(device=dev, dtype=torch.int32).contiguous()

    def _upload(self, voice, dev):
        """The fs2_acoustic_voices of this phase: the voices' structs (their per-call position pointers included) uploaded from a
        fresh pinned block with one non_blocking copy (the caching host allocator keeps the block until the copy is done), and what
        must stay alive while the call is made."""
        structs = [mk._packed[0] for mk in self.models]
        raw = bytearray(b"".join(bytes(m) for m in structs))
        host = torch.empty(len(raw), dtype=torch.uint8, pin_memory=True)
        host.copy_(torch.frombuffer(raw, dtype=torch.uint8))
        table = host.to(dev, non_blocking=True)
        arr = L.acoustic_model_array(structs)
        va = L.AcousticVoices(n=len(structs), models=C.addressof(arr), models_dev=table.data_ptr(), voice=voice.data_ptr())
        return va, (arr, table)

    def _workspace(self, nbytes: int, dev):
        self._ws, self._ws_stream = _streams.workspace((self._ws, self._ws_stream), nbytes, dev, grow=1.25, slack=1024)
        return self._ws
