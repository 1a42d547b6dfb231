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
from .. import packing
from .._modtree import get, populate
from ..spec import fastspeech2_spec, read_dataset_files
from ..synth import sinusoid_table


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
        self._pos_long = {}          # device position tables longer than max_seq_len, keyed by width
        self._ws = None
        self._stats_host = None

    # ------------------------------------------------------------------ packing
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
        tab = self._pos_long.get(width)
        if tab is None or tab.shape[0] < n or tab.device != dev:
            rows = max(2048, 1 << (n - 1).bit_length())
            tab = sinusoid_table(rows, width).to(dev)
            self._pos_long[width] = tab
        return tab.data_ptr(), tab.shape[0]

    def _workspace(self, nbytes: int, dev):
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
            self._ws = torch.empty(int(nbytes * 1.25) + 1024, dtype=torch.uint8, device=dev)
        return self._ws

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, speakers, texts, src_lens, max_src_len, mels=None, mel_lens=None, max_mel_len=None,
                p_targets=None, e_targets=None, d_targets=None, p_control=1.0, e_control=1.0, d_control=1.0, ragged=None):
        """The reference's forward; `ragged` (None: the module's `ragged` attribute) selects the ragged mode described in __init__."""
        # the C ABI sets up per-device kernel attributes for the CURRENT device: make the model's device current
        dev = get(self, "mel_linear.weight").device
        with (torch.cuda.device(dev) if dev.type == "cuda" else contextlib.nullcontext()):
            return self._forward(speakers, texts, src_lens, max_src_len, mels, mel_lens, max_mel_len, p_targets, e_targets, d_targets,
                                 p_control, e_control, d_control, self.ragged if ragged is None else bool(ragged))

    def _forward(self, speakers, texts, src_lens, max_src_len, mels=None, mel_lens=None, max_mel_len=None,
                 p_targets=None, e_targets=None, d_targets=None, p_control=1.0, e_control=1.0, d_control=1.0, ragged=False):
        if self.training:
            raise NotImplementedError("H100-native FastSpeech2 is inference-only: call .eval() (utils/model.py:32)")
        p_frame = self.pitch_feature_level == "frame_level"
        e_frame = self.energy_feature_level == "frame_level"
        lib = L.lib()
        m, _keep, dev = self._packed or self._pack()
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
        if self._stats_host is None:
            self._stats_host = torch.zeros(3, dtype=torch.int32).pin_memory()
        tgt = lambda t: None if t is None else t.to(**f32).contiguous()
        p_t, e_t, d_t = tgt(p_targets), tgt(e_targets), tgt(d_targets)

        m.enc_pos, m.enc_pos_rows = self._position(0, Lmax, m.d_model, dev)
        ws_bytes = lib.fs2_encode_workspace_bytes(C.byref(m), B, Lmax)
        ws = self._workspace(ws_bytes, dev)
        ea = L.EncodeArgs(B=B, L=Lmax, texts=texts.data_ptr(), speakers=L.ptr(speakers_d), src_lens=src_lens32.data_ptr(),
                          p_control=float(p_control), e_control=float(e_control), d_control=float(d_control),
                          p_target=0 if p_frame else L.ptr(p_t), e_target=0 if e_frame else L.ptr(e_t), d_target=L.ptr(d_t),
                          p_pred=0 if p_frame else p_pred.data_ptr(), e_pred=0 if e_frame else e_pred.data_ptr(), logd_pred=logd.data_ptr(),
                          d_rounded=d_rounded.data_ptr(), mel_lens=mel_lens_out.data_ptr(), mel_lens32=mel_lens32.data_ptr(),
                          cum_dur=cum.data_ptr(), x_adapted=x_adapted.data_ptr(), len_stats=stats_dev.data_ptr(),
                          len_stats_host=self._stats_host.data_ptr(), workspace=ws.data_ptr(), workspace_bytes=ws.numel())
        encode = lib.fs2_acoustic_encode_ragged if ragged else lib.fs2_acoustic_encode
        L.check(encode(C.byref(m), C.byref(ea), stream), "fs2_acoustic_encode")

        if max_mel_len is not None:
            T = int(max_mel_len)
        else:
            # the one unavoidable host sync: the output shape depends on the predicted durations (utils/tools.py:94)
            torch.cuda.current_stream(dev).synchronize()
            T = int(self._stats_host[0])
            if int(self._stats_host[2]) != 0:
                raise L.Fs2Error(f"{int(self._stats_host[2])} predicted durations are NaN / inf / > 1e6 frames "
                                 "(the reference raises on them too, model/modules.py:186)")
        if T <= 0:
            raise L.Fs2Error("all predicted durations are zero: nothing to decode")
        if mel_lens is not None and d_targets is not None:
            mask_lens32 = mel_lens.to(device=dev, dtype=torch.int32).contiguous()   # teacher forcing: the caller's mask (fastspeech2.py:60-64)
        else:
            mask_lens32 = mel_lens32       # free-running: the adaptor rebuilds the mask from the predicted lengths (modules.py:132-137)

        m.dec_pos, m.dec_pos_rows = self._position(1, T, m.d_model, dev)
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
        ws_bytes = lib.fs2_decode_workspace_bytes(C.byref(m), B, T)
        ws = self._workspace(ws_bytes, dev)
        da = L.DecodeArgs(B=B, L=Lmax, T=T, x_adapted=x_adapted.data_ptr(), cum_dur=cum.data_ptr(),
                          mel_mask_lens=mask_lens32.data_ptr(), p_control=float(p_control),
                          p_target_frames=L.ptr(p_t) if p_frame else 0, e_target_frames=L.ptr(e_t) if e_frame else 0,
                          p_pred_frames=p_pred.data_ptr() if p_frame else 0, e_pred_frames=e_pred.data_ptr() if e_frame else 0,
                          mel=mel.data_ptr(), postnet_mel=post.data_ptr(),
                          workspace=ws.data_ptr(), workspace_bytes=ws.numel())
        decode = lib.fs2_acoustic_decode_ragged if ragged else lib.fs2_acoustic_decode
        L.check(decode(C.byref(m), C.byref(da), stream), "fs2_acoustic_decode")

        src_masks = torch.arange(Lmax, device=dev)[None, :] >= src_lens32[:, None]
        mel_masks = torch.arange(T, device=dev)[None, :] >= mask_lens32[:, None]
        return (mel, post, p_pred, e_pred, logd, d_targets if d_targets is not None else d_rounded,
                src_masks, mel_masks, src_lens_in, mel_lens_out)
