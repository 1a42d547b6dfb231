"""ctypes binding of libfs2b200.so (the C ABI in include/fs2b200.h).

There is NO fallback: if the shared library is missing or a call fails, this raises.  The product
path never routes through PyTorch ops or the CPU oracle for compute.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfs2b200.so")

ABI_VERSION = 11
MAX_LAYERS, MAX_POSTNET, MAX_STAGES, MAX_RESBLOCKS, MAX_DIL = 12, 8, 8, 32, 4
ACT_NONE, ACT_RELU, ACT_TANH, ACT_LRELU = 0, 1, 2, 3
CONV_AUTO, CONV_SIMT, CONV_TC = 0, 1, 2
TC_ENCODER, TC_PREDICTORS, TC_DECODER, TC_POSTNET = 1, 2, 4, 8
TC_DECODER_F8, TC_POSTNET_F8 = 16, 32
TC_VARIANT_F8 = 1
TC_VARIANT_NB64 = 2
TC_VARIANT_SEGMENTED = 4
PROF_CLASSES = 5

fp = C.c_void_p   # device pointers travel as integers (tensor.data_ptr())
i32, i64, f32 = C.c_int, C.c_int64, C.c_float


class Conv1dArgs(C.Structure):
    _fields_ = [("x", fp), ("x_batch_stride", i64), ("x_row_stride", i64),
                ("B", i32), ("T", i32), ("Cin", i32),
                ("w", fp), ("bias", fp),
                ("N", i32), ("taps", i32), ("dilation", i32), ("pad_left", i32),
                ("w_tc", fp), ("backend", i32), ("tc_variant", C.c_uint),
                ("in_act", i32), ("in_slope", f32), ("out_act", i32), ("out_slope", f32),
                ("res", fp), ("res_batch_stride", i64), ("res_row_stride", i64),
                ("alpha", f32), ("accumulate", i32),
                ("row_lens", fp),
                ("y", fp), ("y_batch_stride", i64), ("y_row_stride", i64),
                ("x_lens", fp), ("lens_scale", i32)]


class LayerNormArgs(C.Structure):
    _fields_ = [("x", fp), ("y", fp), ("B", i32), ("T", i32), ("C", i32),
                ("gamma", fp), ("beta", fp), ("eps", f32), ("row_lens", fp), ("pre_relu", i32)]


class AttentionArgs(C.Structure):
    _fields_ = [("qkv", fp), ("ctx", fp), ("B", i32), ("T", i32), ("H", i32), ("Dh", i32),
                ("key_lens", fp), ("scale", f32), ("backend", i32), ("workspace", fp), ("workspace_bytes", C.c_size_t)]


class EmbedArgs(C.Structure):
    _fields_ = [("ids", fp), ("table", fp), ("pos", fp), ("y", fp), ("B", i32), ("L", i32), ("D", i32), ("n_vocab", i32)]


class RowBiasArgs(C.Structure):
    _fields_ = [("x", fp), ("table", fp), ("idx", fp), ("B", i32), ("L", i32), ("D", i32), ("n_rows", i32)]


class VarianceHeadArgs(C.Structure):
    _fields_ = [("h", fp), ("w", fp), ("b", fp), ("B", i32), ("L", i32), ("C", i32),
                ("lens", fp), ("control", f32), ("target", fp),
                ("bins", fp), ("n_edges", i32), ("emb", fp), ("D", i32), ("x", fp),
                ("pred_out", fp)]


class DurationsArgs(C.Structure):
    _fields_ = [("src", fp), ("use_target", i32), ("d_control", f32), ("B", i32), ("L", i32),
                ("d_rounded", fp), ("cum", fp), ("mel_lens", fp), ("mel_lens32", fp), ("len_stats", fp)]


class LengthRegulateArgs(C.Structure):
    _fields_ = [("x", fp), ("cum", fp), ("pos", fp), ("y", fp), ("B", i32), ("L", i32), ("T", i32), ("D", i32)]


class ConvPostArgs(C.Structure):
    _fields_ = [("x", fp), ("B", i32), ("T", i32), ("C", i32), ("w", fp), ("bias", fp), ("taps", i32),
                ("in_slope", f32), ("wav", fp), ("lens", fp), ("lens_scale", i32)]


class FftBlockWeights(C.Structure):
    _fields_ = [(n, fp) for n in ("w_qkv", "b_qkv", "w_o", "b_o", "ln1_g", "ln1_b", "w_1", "b_1", "w_2", "b_2", "ln2_g", "ln2_b",
                                  "w_qkv_tc", "w_o_tc", "w_1_tc", "w_2_tc")]


class PredictorWeights(C.Structure):
    _fields_ = [(n, fp) for n in ("w_c1", "b_c1", "ln1_g", "ln1_b", "w_c2", "b_c2", "ln2_g", "ln2_b", "w_out", "b_out", "w_c1_tc", "w_c2_tc")]


class AcousticModel(C.Structure):
    _fields_ = [("d_model", i32), ("n_head", i32), ("d_inner", i32), ("k1", i32), ("k2", i32), ("n_enc", i32), ("n_dec", i32),
                ("n_mel", i32), ("vp_filter", i32), ("vp_kernel", i32), ("n_bins", i32), ("n_vocab", i32), ("n_speakers", i32),
                ("enc_pos_rows", i32), ("dec_pos_rows", i32), ("tc_mask", i32),
                ("pitch_frame_level", i32), ("energy_frame_level", i32),
                ("word_emb", fp), ("enc_pos", fp), ("dec_pos", fp), ("spk_emb", fp),
                ("enc", FftBlockWeights * MAX_LAYERS), ("dec", FftBlockWeights * MAX_LAYERS),
                ("dur", PredictorWeights), ("pitch", PredictorWeights), ("energy", PredictorWeights),
                ("pitch_bins", fp), ("energy_bins", fp), ("pitch_emb", fp), ("energy_emb", fp),
                ("w_mel", fp), ("b_mel", fp),
                ("n_postnet", i32), ("post_k", i32),
                ("post_cin", i32 * MAX_POSTNET), ("post_cout", i32 * MAX_POSTNET),
                ("w_post", fp * MAX_POSTNET), ("b_post", fp * MAX_POSTNET),
                ("w_mel_tc", fp), ("w_post_tc", fp * MAX_POSTNET)]


class EncodeArgs(C.Structure):
    _fields_ = [("B", i32), ("L", i32), ("texts", fp), ("speakers", fp), ("src_lens", fp),
                ("p_control", f32), ("e_control", f32), ("d_control", f32),
                ("p_target", fp), ("e_target", fp), ("d_target", fp),
                ("p_pred", fp), ("e_pred", fp), ("logd_pred", fp), ("d_rounded", fp),
                ("mel_lens", fp), ("mel_lens32", fp), ("cum_dur", fp), ("x_adapted", fp),
                ("len_stats", fp), ("len_stats_host", fp),
                ("workspace", fp), ("workspace_bytes", C.c_size_t)]


class DecodeArgs(C.Structure):
    _fields_ = [("B", i32), ("L", i32), ("T", i32), ("x_adapted", fp), ("cum_dur", fp), ("mel_mask_lens", fp),
                ("p_control", f32), ("p_target_frames", fp), ("e_target_frames", fp), ("p_pred_frames", fp), ("e_pred_frames", fp),
                ("mel", fp), ("postnet_mel", fp), ("workspace", fp), ("workspace_bytes", C.c_size_t)]


class VocoderModel(C.Structure):
    _fields_ = [("n_mel", i32), ("c0", i32), ("n_stages", i32), ("n_kernels", i32), ("n_dil", i32),
                ("rates", i32 * MAX_STAGES), ("up_k", i32 * MAX_STAGES),
                ("rb_k", i32 * (MAX_DIL + 4)), ("rb_dil", (i32 * MAX_DIL) * (MAX_DIL + 4)),
                ("w_pre", fp), ("b_pre", fp),
                ("w_up_a", fp * MAX_STAGES), ("w_up_b", fp * MAX_STAGES), ("b_up", fp * MAX_STAGES),
                ("w_rb1", (fp * MAX_DIL) * MAX_RESBLOCKS), ("b_rb1", (fp * MAX_DIL) * MAX_RESBLOCKS),
                ("w_rb2", (fp * MAX_DIL) * MAX_RESBLOCKS), ("b_rb2", (fp * MAX_DIL) * MAX_RESBLOCKS),
                ("w_post", fp), ("b_post", fp),
                ("w_pre_tc", fp), ("w_up_a_tc", fp * MAX_STAGES), ("w_up_b_tc", fp * MAX_STAGES),
                ("w_rb1_tc", (fp * MAX_DIL) * MAX_RESBLOCKS), ("w_rb2_tc", (fp * MAX_DIL) * MAX_RESBLOCKS),
                ("f8_mask", i32), ("fused_mask", i32), ("pair_mask", i32), ("pair_kmax", i32)]


class ResstackArgs(C.Structure):
    _K = MAX_DIL + 4
    _fields_ = [("x", fp), ("y", fp), ("B", i32), ("N", i32), ("C", i32), ("n_kernels", i32), ("n_dil", i32),
                ("k", i32 * (MAX_DIL + 4)), ("dil", (i32 * MAX_DIL) * (MAX_DIL + 4)),
                ("w1_tc", (fp * MAX_DIL) * (MAX_DIL + 4)), ("b1", (fp * MAX_DIL) * (MAX_DIL + 4)),
                ("w2_tc", (fp * MAX_DIL) * (MAX_DIL + 4)), ("b2", (fp * MAX_DIL) * (MAX_DIL + 4)),
                ("alpha", f32), ("accumulate", i32), ("lens", fp), ("lens_scale", i32)]


class WavInt16Args(C.Structure):
    _fields_ = [("wav", fp), ("wav_batch_stride", i64), ("B", i32), ("N", i64), ("lens", fp), ("scale", f32), ("out", fp)]


class VocoderArgs(C.Structure):
    _fields_ = [("B", i32), ("T", i32), ("mel", fp), ("mel_batch_stride", i64), ("mel_row_stride", i64),
                ("wav", fp), ("workspace", fp), ("workspace_bytes", C.c_size_t), ("mel_lens", fp)]


EXPORTS = {
    # name: (restype, argtypes)
    "fs2_abi_version": (i32, []),
    "fs2_kernel_launch_count": (i64, []),
    "fs2_build_info": (C.c_char_p, []),
    "fs2_struct_size": (C.c_size_t, [i32]),
    "fs2_profile_begin": (i32, []),
    "fs2_profile_end": (i32, [C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(i64)]),
    "fs2_conv1d": (i32, [C.POINTER(Conv1dArgs), fp]),
    "fs2_conv_tc_block": (i32, [i32]),
    "fs2_conv_tc_block_f8": (i32, [i32]),
    "fs2_conv_tc_plan": (i32, [C.c_void_p, i32, C.c_void_p]),
    "fs2_layernorm": (i32, [C.POINTER(LayerNormArgs), fp]),
    "fs2_attention": (i32, [C.POINTER(AttentionArgs), fp]),
    "fs2_attention_workspace_bytes": (C.c_size_t, [i32, i32, i32]),
    "fs2_embed_positions": (i32, [C.POINTER(EmbedArgs), fp]),
    "fs2_add_speaker": (i32, [C.POINTER(RowBiasArgs), fp]),
    "fs2_variance_head": (i32, [C.POINTER(VarianceHeadArgs), fp]),
    "fs2_durations": (i32, [C.POINTER(DurationsArgs), fp]),
    "fs2_length_regulate": (i32, [C.POINTER(LengthRegulateArgs), fp]),
    "fs2_conv_post": (i32, [C.POINTER(ConvPostArgs), fp]),
    "fs2_resstack": (i32, [C.POINTER(ResstackArgs), fp]),
    "fs2_wav_to_int16": (i32, [C.POINTER(WavInt16Args), fp]),
    "fs2_resstack_plan": (i32, [C.POINTER(ResstackArgs), i32, C.c_void_p]),
    "fs2_transpose_bct_to_btc": (i32, [fp, fp, i32, i32, i32, fp]),
    "fs2_add_positions": (i32, [fp, fp, i32, i32, i32, fp]),
    "fs2_encode_workspace_bytes": (C.c_size_t, [C.POINTER(AcousticModel), i32, i32]),
    "fs2_acoustic_encode": (i32, [C.POINTER(AcousticModel), C.POINTER(EncodeArgs), fp]),
    "fs2_decode_workspace_bytes": (C.c_size_t, [C.POINTER(AcousticModel), i32, i32]),
    "fs2_acoustic_decode": (i32, [C.POINTER(AcousticModel), C.POINTER(DecodeArgs), fp]),
    "fs2_acoustic_encode_ragged": (i32, [C.POINTER(AcousticModel), C.POINTER(EncodeArgs), fp]),
    "fs2_acoustic_decode_ragged": (i32, [C.POINTER(AcousticModel), C.POINTER(DecodeArgs), fp]),
    "fs2_vocoder_workspace_bytes": (C.c_size_t, [C.POINTER(VocoderModel), i32, i32]),
    "fs2_vocoder_forward": (i32, [C.POINTER(VocoderModel), C.POINTER(VocoderArgs), fp]),
}

_lib = None


class Fs2Error(RuntimeError):
    pass


def lib():
    """Load (once) and return the shared library.  Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Fs2Error(f"{LIB_PATH} not found: run `python -m fastspeech2_b200.build` (or __graft_entry__.build()); "
                           "there is no PyTorch/CPU fallback for the hot path")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in EXPORTS.items():
            fn = getattr(handle, name)      # AttributeError if the symbol is missing
            fn.restype, fn.argtypes = res, args
        if handle.fs2_abi_version() != ABI_VERSION:
            raise Fs2Error(f"ABI mismatch: library {handle.fs2_abi_version()} vs binding {ABI_VERSION}; rebuild")
        _lib = handle
    return _lib


_ERR = {-1: "FS2_ERR_ARG", -2: "FS2_ERR_UNSUPPORTED", -3: "FS2_ERR_WORKSPACE"}


def check(rc: int, what: str = "fs2 call"):
    if rc == 0:
        return
    if rc <= -1000:
        raise Fs2Error(f"{what}: CUDA error {-(rc + 1000)}")
    raise Fs2Error(f"{what}: {_ERR.get(rc, rc)}")


def ptr(t):
    """Device pointer of a tensor (0 for None)."""
    return 0 if t is None else t.data_ptr()
