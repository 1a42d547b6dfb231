/* fs2b200.h -- C ABI of the H100-native FastSpeech2 + HiFi-GAN inference path.
 *
 * The reference (ming024/FastSpeech2) has no FFI: its "plugin API" for this path is two nn.Module
 * classes.  This library is what a native binding underneath those two classes calls:
 *
 *   fs2_acoustic_encode  + fs2_acoustic_decode   replace  model.fastspeech2.FastSpeech2.forward
 *                                                 (model/fastspeech2.py:43-110; split at the one
 *                                                 data-dependent shape, max(mel_len), modules.py:136)
 *   fs2_vocoder_forward                           replaces hifigan.models.Generator.forward
 *                                                 (hifigan/models.py:149-165)
 *
 * plus one entry point per fused operator (used by the model-level calls and by the parity tests):
 *
 *   fs2_embed_positions   transformer/Models.py:89-91        fs2_conv1d        nn.Conv1d / nn.Linear / ConvTranspose1d call sites
 *   fs2_attention         transformer/Modules.py:14-25       fs2_layernorm     nn.LayerNorm + masked_fill (Layers.py:25,28)
 *   fs2_variance_head     model/modules.py:80-100,:246-250   fs2_durations     model/modules.py:132-135,:185-187
 *   fs2_length_regulate   model/modules.py:167-194           fs2_conv_post     hifigan/models.py:161-163
 *
 * Conventions: every pointer is a DEVICE pointer unless named *_host; activations are fp32,
 * channels-last ([B][T][C], C contiguous); the library never allocates, frees or synchronises --
 * the caller provides outputs and a workspace and owns the stream.  Return value: FS2_OK or a
 * negative error; a CUDA launch error e is returned as FS2_ERR_CUDA - e.  No exceptions, no exit().
 */
#ifndef FS2B200_H
#define FS2B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* fs2_stream_t; /* cudaStream_t */

enum {
  FS2_OK = 0,
  FS2_ERR_ARG = -1,         /* null pointer / non-positive size / misaligned pointer */
  FS2_ERR_UNSUPPORTED = -2, /* configuration outside what the kernels specialise on */
  FS2_ERR_WORKSPACE = -3,   /* workspace too small */
  FS2_ERR_CUDA = -1000      /* FS2_ERR_CUDA - cudaError_t */
};

enum { FS2_ACT_NONE = 0, FS2_ACT_RELU = 1, FS2_ACT_TANH = 2, FS2_ACT_LRELU = 3 };
enum { FS2_CONV_AUTO = 0, FS2_CONV_SIMT = 1, FS2_CONV_TC = 2 };
/* which parts of the acoustic model may use the split-FP16 tensor-core kernel (fs2_acoustic_model.tc_mask) */
enum { FS2_TC_ENCODER = 1, FS2_TC_PREDICTORS = 2, FS2_TC_DECODER = 4, FS2_TC_POSTNET = 8,
       /* the decoder's / PostNet's w_*_tc tiles are in the f16+f8 format (see FS2_TC_VARIANT_F8) */
       FS2_TC_DECODER_F8 = 16, FS2_TC_POSTNET_F8 = 32 };
/* fs2_conv1d_args.tc_variant bits.  F8: w_tc holds the two-MMA operand split -- fp16 hi tiles as in the three-MMA split, and in
 * place of the fp16 lo tiles E4M3 tiles [hi * 2^-12 | lo] that one K = 32 E4M3 MMA multiplies with the activations'
 * [lo * 2^12 | hi]: y ~ a_hi.w_hi + (a_lo.w_hi + a_hi.w_lo) with the bracket at E4M3 precision (relative error ~2^-16 instead
 * of ~2^-22; half the tensor-core work of the three-MMA split).  The correction accumulates separately from the main term (Hopper
 * adds E4M3 products with reduced precision), so F8 tiles use NB = fs2_conv_tc_block_f8(N) <= 64 output channels per work item.
 * The correction saturates from |a| = 256 on, not 448: there lo * 2^12 can leave E4M3's range (|lo| up to 2^-3 once the fp16 ulp of
 * a is 2^-2), which costs up to 2^-14 relative (about 12 % of values in [256, 448)); from 448 on hi saturates too.  The shipped
 * HiFi-GAN checkpoints stay below 24 on real mels (tests/test_tc_precision_cpu.py). */
enum { FS2_TC_VARIANT_F8 = 1,
       /* w_tc is tiled for 64 output channels per work item (pack_conv_tc(w, nb=64)): the hi*hi term and the two cross terms then
        * accumulate in separate register accumulators.  Used by the K-segmented encoder / predictor path (see fs2_acoustic_model). */
       FS2_TC_VARIANT_NB64 = 2,
       /* with NB64: w_tc holds taps * (C_in / 256) one-tap tile buffers back to back (packing.pack_conv_tc_segments) and the conv is
        * evaluated K-SEGMENTED inside one launch: every (tile, tap, 256-channel chunk) is a work unit with a fresh 16-step accumulator,
        * the units of a tile run back to back on one CTA and add into y in fp32 round-to-nearest (bias with the first, residual and
        * pad-row mask with the last).  Needs dilation 1, alpha 1, no output activation, C_in % 256 == 0, N % 64 == 0. */
       FS2_TC_VARIANT_SEGMENTED = 4 };

/* Tensor-core weight tiles.  For a conv weight w[taps][Cin][N] with NB = fs2_conv_tc_block(N) output channels per work item
 * (fs2_conv_tc_block_f8(N) for FS2_TC_VARIANT_F8 tiles, whose plane 1 holds the E4M3 [hi * 2^-12 | lo] chunks instead of fp16 lo),
 * s = a per-layer power of two, hi = fp16(s*w), lo = fp16(s*w - hi), the tiled byte buffer is
 *     128-byte header (float32[0] = 1/s)  |  [N/NB][Cin/16][taps][2: hi,lo][2: 16-byte K chunk][NB][8 halfs]
 * i.e. every (K-block, tap) stage is one contiguous 64*NB-byte smem image (no-swizzle K-major, fp16), fetched by one
 * cp.async.bulk.  fastspeech2_b200/packing.py::pack_conv_tc builds it. */
int fs2_conv_tc_block(int N);    /* 0 when N is not supported by the tensor-core kernel */
int fs2_conv_tc_block_f8(int N); /* the same for FS2_TC_VARIANT_F8 tiles: the largest multiple of 16 <= 64 that divides N (N itself if N <= 64) */
struct fs2_conv1d_args;
/* Launch plan of the tensor-core kernel; a work item is one 128-row tile x NG blocks of NB output channels, computed one block after
 * another from the tile's input slab, which stays in shared memory (SA >= C_in / 16 when NG > 1). */
typedef struct fs2_conv_tc_plan_t {
  int32_t NB;              /* output channels per block */
  int32_t TG;              /* accumulators per tile: 1 = all split terms together, 2 = {hi*hi | the cross terms} */
  int32_t SA, SB;          /* activation slab stages, weight stages */
  int32_t TPS;             /* conv taps per weight stage */
  int32_t R;               /* slab rows */
  int32_t acc_regs;        /* accumulator registers per consumer thread */
  int32_t tiles_per_batch; /* 128-row tiles per utterance */
  int32_t n_items, grid;   /* (tile, block) pairs of the padded shape, i.e. NG x the work items; CTAs */
  int32_t smem;            /* dynamic shared memory bytes */
  int32_t NG;              /* channel blocks per work item */
} fs2_conv_tc_plan_t;
/* The plan the tensor-core kernel would use for this call on a device with num_sms SMs (pure host logic, no CUDA call, pointers are
 * only checked for alignment).  Returns FS2_ERR_UNSUPPORTED for shapes the kernel does not take. */
int fs2_conv_tc_plan(const struct fs2_conv1d_args* a, int num_sms, fs2_conv_tc_plan_t* out);
/* Tile of the exact fp32 kernel (FS2_CONV_SIMT). */
typedef struct fs2_conv_simt_plan_t {
  int32_t BM;              /* rows per CTA: 64 or 128 */
  int32_t BN;              /* output channels per CTA: 32, 64 or 128 */
  int32_t grid_x, grid_y;
} fs2_conv_simt_plan_t;
/* The tile the exact kernel would use for this call on a device with num_sms SMs (pure host logic, no CUDA call, pointers are not
 * read).  Returns FS2_ERR_ARG / FS2_ERR_UNSUPPORTED for shapes the kernel does not take. */
int fs2_conv_simt_plan(const struct fs2_conv1d_args* a, int num_sms, fs2_conv_simt_plan_t* out);

#define FS2_MAX_LAYERS 12
#define FS2_MAX_POSTNET 8
#define FS2_MAX_STAGES 8
#define FS2_MAX_RESBLOCKS 32
#define FS2_MAX_DIL 4

/* ------------------------------------------------------------------ operators */

/* y[b,t,n] = (accumulate ? y : 0) + alpha * ( out_act( bias[n] + sum_{j<taps} sum_c in_act(x[b, t + j*dilation - pad_left, c]) * w[j][c][n] ) + res[b,t,n] )
 * rows outside [0,T) read as zero (Conv1d zero padding); rows t >= row_lens[b] are written as exact 0 when row_lens != NULL.
 * Strides are in elements.  Covers nn.Linear (taps=1), nn.Conv1d (any odd k, dilation), and one phase group of
 * ConvTranspose1d (two taps, y_row_stride = u*C_out; see fs2_vocoder_model).
 * Both kernels: pointers 16-byte aligned, strides % 4 == 0; the exact kernel Cin % 16 == 0 or Cin == 8 (HiFi-GAN V2's last stage), the
 * tensor-core kernel Cin % 16 == 0.  The tensor-core kernel additionally needs w_tc,
 * N % 16 == 0, x 32-byte aligned with x strides % 8 == 0 (256-bit loads), in_act in {NONE, LRELU with 0 <= slope <= 1} and
 * (taps-1)*dilation <= 256; anything else is served by the exact kernel under FS2_CONV_AUTO and refused (FS2_ERR_UNSUPPORTED)
 * under FS2_CONV_TC.  Activations beyond +-65504 saturate in the fp16 hi/lo split of the tensor-core kernel. */
typedef struct fs2_conv1d_args {
  const float* x; int64_t x_batch_stride, x_row_stride;
  int B, T, Cin;
  const float* w;    /* [taps][Cin][N] */
  const float* bias; /* [N] or NULL */
  int N, taps, dilation, pad_left;
  const float* w_tc; /* NULL, or the same weights in the tensor-core tile layout (see "tensor-core weight tiles" below) */
  int backend;       /* FS2_CONV_AUTO: split-FP16 tensor-core kernel when w_tc is given and the shape qualifies, else the fp32 CUDA-core kernel */
  unsigned tc_variant; /* FS2_TC_VARIANT_* bits describing the format of w_tc */
  int in_act; float in_slope;
  int out_act; float out_slope;
  const float* res; int64_t res_batch_stride, res_row_stride; /* NULL = none */
  float alpha; int accumulate;
  const int32_t* row_lens; /* [B] or NULL */
  float* y; int64_t y_batch_stride, y_row_stride;
  /* Ragged batch: NULL, or [B] per-utterance lengths.  Utterance b then has n_b = clamp(x_lens[b] * lens_scale, 0, T) rows: input rows
   * t >= n_b read as zero (as rows outside [0, T) do), output rows t >= n_b are unspecified (row_lens still zeroes rows >= row_lens[b]
   * where they are written), and no work item lying wholly at or beyond n_b runs -- so utterance b is computed exactly as a B = 1 call
   * on its first n_b rows.  lens_scale (rows per length unit, e.g. 256 when x_lens holds mel frames and the rows are audio samples)
   * must be >= 1 when x_lens is given (FS2_ERR_ARG before any CUDA call).  The tensor-core kernel's grid is still sized from the padded
   * shape (the host never reads device lengths); CTAs left without work exit. */
  const int32_t* x_lens; int lens_scale;
} fs2_conv1d_args;
int fs2_conv1d(const fs2_conv1d_args* a, fs2_stream_t stream);

/* y = LayerNorm_C(x or relu(x)) * gamma + beta over the last dim, then rows t >= row_lens[b] := 0.  x,y contiguous [B][T][C]; C%4==0, C<=1024. */
typedef struct fs2_layernorm_args {
  const float* x; float* y; int B, T, C;
  const float* gamma; const float* beta; float eps;
  const int32_t* row_lens; /* [B] or NULL */
  int pre_relu;            /* 1: LayerNorm(relu(x)) -- the predictors' conv -> ReLU -> LayerNorm (model/modules.py:242-250) when the conv left its ReLU to this op */
} fs2_layernorm_args;
int fs2_layernorm(const fs2_layernorm_args* a, fs2_stream_t stream);

/* ctx[b,t,h*Dh+j] = sum_s softmax_s( q[b,t,h,:].k[b,s,h,:] * scale , keys s >= key_lens[b] masked ) * v[b,s,h,j]
 * qkv: [B][T][3*H*Dh] rows laid out q|k|v, heads contiguous inside each.  Dh must be 128.  Query rows t >= key_lens[b] are written as 0
 * (the reference zeroes them after the following LayerNorm, transformer/Layers.py:25). */
typedef struct fs2_attention_args {
  const float* qkv; float* ctx; int B, T, H, Dh;
  const int32_t* key_lens; float scale;
  int backend;                  /* 0 = exact fp32 flash-style kernel; 2 = ONE fused tensor-core kernel (QK^T, softmax, PV; scores stay in
                                   registers, any T).  Any other value: FS2_ERR_ARG */
  void* workspace; size_t workspace_bytes;   /* backend 2: >= fs2_attention_workspace_bytes(B, T, H) bytes; backend 0 ignores it */
} fs2_attention_args;
int fs2_attention(const fs2_attention_args* a, fs2_stream_t stream);
size_t fs2_attention_workspace_bytes(int B, int T, int H);

/* y[b,l,:] = table[ids[b,l]] + pos[l]   (the speaker embedding is added separately, by fs2_add_speaker) */
typedef struct fs2_embed_args {
  const int64_t* ids; const float* table; const float* pos; float* y; int B, L, D, n_vocab;
} fs2_embed_args;
int fs2_embed_positions(const fs2_embed_args* a, fs2_stream_t stream);

/* x[b,l,:] += table[idx[b]]  for every l < L (padded rows included, model/fastspeech2.py:68-71) */
typedef struct fs2_rowbias_args { float* x; const float* table; const int64_t* idx; int B, L, D, n_rows; } fs2_rowbias_args;
int fs2_add_speaker(const fs2_rowbias_args* a, fs2_stream_t stream);

/* pred[b,l] = (h[b,l,:].w + *b), 0 where l >= lens[b]; if bins != NULL:
 *   v = target ? target[b,l] : pred*control (pred_out then holds the scaled value),  i = #edges < v (torch.bucketize right=False:
 *   -inf -> 0, +inf -> #edges < inf, NaN -> n_edges, as ATen's search picks),  x[b,l,:] += emb[i]. */
typedef struct fs2_variance_head_args {
  const float* h; const float* w; const float* b; int B, L, C;
  const int32_t* lens; float control; const float* target;
  const float* bins; int n_edges; const float* emb; int D; float* x;
  float* pred_out;
} fs2_variance_head_args;
int fs2_variance_head(const fs2_variance_head_args* a, fs2_stream_t stream);

/* d = use_target ? src[b,l] : clamp(rint(exp(src[b,l]) - 1) * d_control, min=0) (torch.clamp: NaN stays NaN, so d_rounded holds NaN
 * where the reference's does); reps = max((int)d, 0);
 * cum[b,l] = inclusive prefix sum of reps; mel_lens[b] = cum[b,L-1]; len_stats[0] = max_b mel_lens, [1] = sum_b mel_lens,
 * [2] = number of NaN / +-inf / > 1e6 durations (those contribute 0 frames; the reference's int() raises on them).  The call zeroes
 * len_stats. */
typedef struct fs2_durations_args {
  const float* src; int use_target; float d_control; int B, L;
  float* d_rounded;     /* [B][L] or NULL */
  int32_t* cum;         /* [B][L] */
  int64_t* mel_lens;    /* [B] */
  int32_t* mel_lens32;  /* [B] or NULL */
  int32_t* len_stats;   /* [3] */
} fs2_durations_args;
int fs2_durations(const fs2_durations_args* a, fs2_stream_t stream);

/* y[b,t,:] = (t < cum[b,L-1] ? x[b, upper_bound(cum[b,:], t), :] : 0) + (pos ? pos[t,:] : 0),  t < T */
typedef struct fs2_length_regulate_args {
  const float* x; const int32_t* cum; const float* pos; float* y; int B, L, T, D;
} fs2_length_regulate_args;
int fs2_length_regulate(const fs2_length_regulate_args* a, fs2_stream_t stream);

/* wav[b,t] = tanh( *bias + sum_{j<taps} sum_c lrelu_slope(x[b,t+j-pad,c]) * w[j][c] )   (hifigan/models.py:161-163)
 * lens: NULL, or [B] per-utterance lengths with n_b = clamp(lens[b] * lens_scale, 0, T) (lens_scale >= 1, else FS2_ERR_ARG): rows
 * t >= n_b of x read as zero and wav[b,t] = 0 exactly for t >= n_b, i.e. each utterance is the waveform of a B = 1 call on its first
 * n_b rows followed by silence. */
typedef struct fs2_conv_post_args {
  const float* x; int B, T, C; const float* w; const float* bias; int taps; float in_slope; float* wav;
  const int32_t* lens; int lens_scale;
} fs2_conv_post_args;
int fs2_conv_post(const fs2_conv_post_args* a, fs2_stream_t stream);

/* HiFi-GAN multi-receptive-field ResBlock group of one upsample stage as ONE persistent kernel (hifigan/models.py:154-160, ResBlock.forward
 * :96-103):   y = (1/n_kernels) * sum_j R_j(x),   R_j: x <- conv_{k_j,1}( lrelu( conv_{k_j,dil_jd}( lrelu(x) ) + b1 ) ) + b2 + x  for d = 0..n_dil-1,
 * lrelu slope 0.1, "same" zero padding at the utterance ends.  x, y: contiguous [B][N][C], C in {8, 16, 32, 64} (the 64- to 8-channel
 * stages of HiFi-GAN V1 and V2; the vocoder also runs 128-channel pairs on the same body, see fs2_vocoder_model::pair_mask); every intermediate stays in shared memory / registers (halo recompute), weights are the f16+f8 tiles of
 * the per-layer kernel (FS2_TC_VARIANT_F8 with N = C: pack_conv_tc(w, f8=True)).  C = 8 is computed as 16 channels whose upper 8 are
 * zero: its weights are the f8 tiles of the conv zero-padded to 16 x 16 (packing.pack_conv_tc_pad16), while x and y stay [B][N][8] and
 * no byte of y outside them is written.  (k-1)*dil/2 <= 32 per conv.  Other shapes: FS2_ERR_UNSUPPORTED.
 * x and y must not overlap (work items re-read halo rows of x): FS2_ERR_ARG. */
typedef struct fs2_resstack_args {
  const float* x; float* y; int B, N, C;
  int n_kernels, n_dil;
  int k[FS2_MAX_DIL + 4]; int dil[FS2_MAX_DIL + 4][FS2_MAX_DIL];
  const float *w1_tc[FS2_MAX_DIL + 4][FS2_MAX_DIL], *b1[FS2_MAX_DIL + 4][FS2_MAX_DIL];   /* dilated conv of each pair */
  const float *w2_tc[FS2_MAX_DIL + 4][FS2_MAX_DIL], *b2[FS2_MAX_DIL + 4][FS2_MAX_DIL];   /* dilation-1 conv of each pair */
  float alpha;     /* weight of every kernel size's result; <= 0: 1/n_kernels (the mean) */
  int accumulate;  /* 1: y += ... (also for the first kernel size) instead of y = ...; with n_kernels = n_dil = 1 the call is ONE fused
                      conv pair  y (+)= alpha * (conv_k,1(lrelu(conv_k,d(lrelu(x)))) + x)  -- the per-pair mode of the 64-channel stage */
  /* Ragged batch: NULL, or [B] per-utterance lengths, n_b = clamp(lens[b] * lens_scale, 0, N) rows (lens_scale >= 1, else FS2_ERR_ARG):
   * rows >= n_b of x read as zero and every conv pads at row n_b, rows >= n_b of y are unspecified, and only the work items that
   * hold a row < n_b run.  The grid is sized from the padded shape (fs2_resstack_plan does not read lengths); CTAs without work exit. */
  const int32_t* lens; int lens_scale;
} fs2_resstack_args;
int fs2_resstack(const fs2_resstack_args* a, fs2_stream_t stream);
/* Launch plan of fs2_resstack; a work item is one slab of MT * 128 rows: TILE output rows with H halo rows at each end. */
typedef struct fs2_resstack_plan_t {
  int32_t MT;              /* 128-row tiles per slab */
  int32_t H;               /* halo rows per side */
  int32_t TILE;            /* output rows per work item */
  int32_t n_items, grid;   /* work items (of the padded shape), CTAs */
  int32_t SB;              /* weight ring stages */
  int32_t smem;            /* dynamic shared memory bytes */
  int32_t acc_regs;        /* accumulator registers per consumer thread */
  int32_t OBOX, n_oboxes;  /* rows per output TMA box, output boxes per tile */
  int32_t TPS;             /* conv taps per weight stage */
} fs2_resstack_plan_t;
/* The plan fs2_resstack would use for this call on a device with num_sms SMs (pure host logic, no CUDA call, pointers are not read). */
int fs2_resstack_plan(const fs2_resstack_args* a, int num_sms, fs2_resstack_plan_t* out);

/* out[b,t] = t < lens[b] ? (int16) trunc(wav[b,t] * scale) : 0   -- the device half of utils.model.vocoder_infer (utils/model.py:82-90:
 * `(wavs.cpu().numpy() * max_wav_value).astype("int16")` then `wavs[i][:lengths[i]]`): 2 bytes per sample cross PCIe instead of 4, the
 * trim is fused, and the copy can be asynchronous.  lens (samples, int64, device) may be NULL.  Values beyond int16 are clamped. */
typedef struct fs2_wav_int16_args {
  const float* wav; int64_t wav_batch_stride; int B; int64_t N;
  const int64_t* lens; float scale; int16_t* out; /* [B][N] contiguous */
} fs2_wav_int16_args;
int fs2_wav_to_int16(const fs2_wav_int16_args* a, fs2_stream_t stream);

/* x[b,t,:] += pos[t,:]   (decoder position add when the length regulator could not fuse it: frame-level variance configs) */
int fs2_add_positions(float* x, const float* pos, int B, int T, int D, fs2_stream_t stream);

/* out[b,t,c] = in[b,c,t]  (mel [B,80,T] -> channels-last) */
int fs2_transpose_bct_to_btc(const float* in, float* out, int B, int C, int T, fs2_stream_t stream);

/* ------------------------------------------------------------------ acoustic model (FastSpeech2.forward) */

typedef struct fs2_fft_block_weights {
  const float *w_qkv, *b_qkv;   /* [D][3D], [3D]   (w_qs|w_ks|w_vs transposed and concatenated) */
  const float *w_o, *b_o;       /* [D][D]          (fc) */
  const float *ln1_g, *ln1_b;
  const float *w_1, *b_1;       /* [k1][D][F]      (pos_ffn.w_1) */
  const float *w_2, *b_2;       /* [k2][F][D] */
  const float *ln2_g, *ln2_b;
  const float *w_qkv_tc, *w_o_tc, *w_1_tc, *w_2_tc; /* tensor-core tiles of the four weights, or NULL */
} fs2_fft_block_weights;

typedef struct fs2_predictor_weights {
  const float *w_c1, *b_c1, *ln1_g, *ln1_b; /* [k][D][F] */
  const float *w_c2, *b_c2, *ln2_g, *ln2_b; /* [k][F][F] */
  const float *w_out, *b_out;               /* [F], [1] */
  const float *w_c1_tc, *w_c2_tc;           /* tensor-core tiles of the two convs (three-MMA split format), or NULL */
} fs2_predictor_weights;

/* Encoder / predictors on the tensor cores (tc_mask bits FS2_TC_ENCODER / FS2_TC_PREDICTORS): these layers feed the discrete duration and
 * pitch / energy bucket decisions, where the truncating tensor-core accumulator of a long K loop (432 accumulation steps for the k = 9
 * conv) costs 5x the error of the fp32 CUDA-core kernel (scripts/flip_census.py).  They therefore run K-SEGMENTED: every
 * (tap, 256-input-channel) slice is its own launch of 16 K-steps whose hi*hi term has its own accumulator (FS2_TC_VARIANT_NB64), and the
 * slices are summed in fp32 round-to-nearest by the epilogue's accumulate path.  Their w_*_tc pointers then hold
 * taps * (C_in / 256) tile buffers back to back (segment (tap, kc) at index tap * (C_in/256) + kc, each 128 + 1024 * N bytes:
 * packing.pack_conv_tc_segments). */
typedef struct fs2_acoustic_model {
  int d_model, n_head, d_inner, k1, k2, n_enc, n_dec, n_mel;
  int vp_filter, vp_kernel, n_bins, n_vocab, n_speakers;
  int enc_pos_rows, dec_pos_rows;            /* rows available in the position tables */
  int tc_mask;                               /* FS2_TC_* bits; parts not selected run the fp32 CUDA-core kernels */
  int pitch_frame_level, energy_frame_level; /* 0 = phoneme-level predictor (before the length regulator), 1 = frame-level (after it): model/modules.py:117-126 vs :139-148 */
  const float *word_emb, *enc_pos, *dec_pos, *spk_emb;
  fs2_fft_block_weights enc[FS2_MAX_LAYERS], dec[FS2_MAX_LAYERS];
  fs2_predictor_weights dur, pitch, energy;
  const float *pitch_bins, *energy_bins, *pitch_emb, *energy_emb;
  const float *w_mel, *b_mel;                /* [D][n_mel] */
  int n_postnet, post_k;
  int post_cin[FS2_MAX_POSTNET], post_cout[FS2_MAX_POSTNET];
  const float *w_post[FS2_MAX_POSTNET], *b_post[FS2_MAX_POSTNET]; /* BatchNorm folded in: [k][cin][cout] */
  const float *w_mel_tc, *w_post_tc[FS2_MAX_POSTNET];             /* tensor-core tiles or NULL */
} fs2_acoustic_model;

/* Phase 1: encoder + speaker add + variance adaptor up to the duration prefix sums. */
typedef struct fs2_encode_args {
  int B, L;
  const int64_t* texts;      /* [B][L] */
  const int64_t* speakers;   /* [B] (ignored when the model has no speaker table) */
  const int32_t* src_lens;   /* [B] */
  float p_control, e_control, d_control;
  const float *p_target, *e_target, *d_target; /* [B][L] or NULL */
  float *p_pred, *e_pred, *logd_pred, *d_rounded; /* [B][L] outputs (d_rounded unused with d_target) */
  int64_t* mel_lens;         /* [B] */
  int32_t* mel_lens32;       /* [B] */
  int32_t* cum_dur;          /* [B][L] */
  float* x_adapted;          /* [B][L][D]: input of the length regulator */
  int32_t* len_stats;        /* device [3]: max and sum of mel_lens, count of NaN / +-inf / > 1e6 durations */
  int32_t* len_stats_host;   /* pinned host [3] or NULL: async D2H copy is enqueued on the stream */
  void* workspace; size_t workspace_bytes;
} fs2_encode_args;
size_t fs2_encode_workspace_bytes(const fs2_acoustic_model* m, int B, int L);
int fs2_acoustic_encode(const fs2_acoustic_model* m, const fs2_encode_args* a, fs2_stream_t stream);

/* Phase 2: length regulator + decoder + mel_linear + PostNet (+ residual). */
typedef struct fs2_decode_args {
  int B, L, T;
  const float* x_adapted; const int32_t* cum_dur;
  const int32_t* mel_mask_lens;  /* [B]: rows t >= len are padding for the decoder masks */
  float p_control;               /* used by frame-level pitch AND energy (the reference passes p_control to both, modules.py:146) */
  const float *p_target_frames, *e_target_frames; /* [B][T] or NULL (frame-level configs, teacher forcing) */
  float *p_pred_frames, *e_pred_frames;           /* [B][T] outputs, required for the predictors configured frame-level */
  float* mel; float* postnet_mel; /* [B][T][n_mel] */
  void* workspace; size_t workspace_bytes;
} fs2_decode_args;
size_t fs2_decode_workspace_bytes(const fs2_acoustic_model* m, int B, int T);
int fs2_acoustic_decode(const fs2_acoustic_model* m, const fs2_decode_args* a, fs2_stream_t stream);

/* Ragged mode of the pair above: same models, arguments and workspace sizes.  Utterance b is bounded by src_lens[b] phonemes in the
 * encoder and the predictors and by mel_mask_lens[b] frames in the decoder, so it is computed exactly -- bit for bit -- as a B = 1
 * call of fs2_acoustic_encode / fs2_acoustic_decode with L = src_lens[b] and T = mel_mask_lens[b] on its own inputs would compute it:
 *   - no value at or beyond an utterance's length (token ids, targets, durations, whatever the workspace holds) reaches its valid
 *     outputs, and no work item lying wholly in the padding is computed (every conv gets the lengths as x_lens);
 *   - p_pred / e_pred / logd_pred / d_rounded / cum_dur are valid on the first src_lens[b] columns (frame-level predictions: on the
 *     first mel_mask_lens[b]); d_rounded is 0 beyond, durations beyond src_lens[b] count as 0 frames;
 *   - mel and postnet_mel are exact zeros in rows >= mel_mask_lens[b];
 *   - x_adapted rows at or beyond src_lens[b] are unspecified;
 *   - the decoder's attention picks its backend per utterance as a B = 1 call would: the fused tensor-core kernel for utterances of
 *     >= 128 frames, the exact kernel for shorter ones.
 * Device lengths are clamped to [0, L] / [0, T] and never read by the host; position-table rows are shared by all utterances. */
int fs2_acoustic_encode_ragged(const fs2_acoustic_model* m, const fs2_encode_args* a, fs2_stream_t stream);
int fs2_acoustic_decode_ragged(const fs2_acoustic_model* m, const fs2_decode_args* a, fs2_stream_t stream);

/* Per-utterance / per-phoneme controls (model/modules.py:85,96,132-135 broadcast `prediction * control`): device fp32 arrays that
 * replace the scalar p_control / d_control of the phase's args where their pointer is set.  Strides are in elements, >= 0 (0 along a
 * broadcast dimension; a negative stride is FS2_ERR_ARG).  48 bytes; the binding pins that size (it is not in fs2_struct_size).
 *   p: pitch AND energy (modules.py:124), c[b, l] with l = phoneme (encode: [B][L] predictions) or frame (decode: frame-level
 *      predictions on [B][T]); not read where the predictor is given its target.
 *   d: durations, encode only, c[b, l] scales round(exp(logd) - 1) before the clamp and int() truncation; not read with d_target. */
typedef struct fs2_control_args {
  const float* p; int64_t p_stride_b, p_stride_l;
  const float* d; int64_t d_stride_b, d_stride_l;
} fs2_control_args;
/* fs2_acoustic_{encode,decode} (ragged = 0) and fs2_acoustic_{encode,decode}_ragged (ragged = 1; other values: FS2_ERR_ARG) with
 * controls.  ctl == NULL, or both pointers NULL: exactly the call without controls (those four entry points are this call).  In ragged
 * mode utterance b with its slice of the controls equals its B = 1 call with c[b:b+1, :src_lens[b]] (frames: :mel_mask_lens[b]), and
 * control columns at or beyond src_lens[b] (frames at or beyond mel_mask_lens[b]) are never read.  A control array holding fp32(c)
 * gives the scalar c's results bit for bit.  Same workspace sizes as the calls without controls. */
int fs2_acoustic_encode_ctl(const fs2_acoustic_model* m, const fs2_encode_args* a, const fs2_control_args* ctl, int ragged,
                            fs2_stream_t stream);
int fs2_acoustic_decode_ctl(const fs2_acoustic_model* m, const fs2_decode_args* a, const fs2_control_args* ctl, int ragged,
                            fs2_stream_t stream);

/* Utterances of several voices in one call: fs2_acoustic_{encode,decode}_ctl, but utterance b runs on voice voice[b] of models[0 .. n):
 * one FastSpeech2 checkpoint per voice, all of one config (fine-tuned copies, or voices trained apart).  The call plans once, on models[0]:
 * its launches, grids and launch count are those of the single-model call at the same B, L and T, and every launch reads each weight
 * and table -- convs, LayerNorms, word / speaker / pitch / energy embeddings, bins, position tables -- from the utterance's own voice.
 * So utterance b equals models[voice[b]] called alone on the same batch, bit for bit: in ragged mode, as that voice's ragged call on its
 * own slice; padded, as row b of that voice's call on the whole batch (no kernel mixes batch rows).
 *   - models_dev: a device copy of the n structs models points at; the kernels read each weight's pointer from models_dev[voice[b]], so
 *     it must stay equal to the host array while the call runs (each voice's per-call position pointers included);
 *   - the host never reads voice: each phase's first launch stages it into the workspace clamped to voice 0, with a validity flag; an
 *     utterance whose voice[b] lies outside [0, n) gets 0 frames (mel_lens[b] = 0, d_rounded[b] = 0) without changing the others, and
 *     its other outputs are unspecified;
 *   - FS2_ERR_ARG before any CUDA call for n outside [1, FS2_MAX_VOICES], a NULL models, models_dev, voice or model, ragged not 0 or 1,
 *     a voice whose position tables have fewer than L (encode) or T (decode) rows, and a model whose layout differs from models[0]'s:
 *     every int field (widths, layers, kernels, n_bins, n_vocab, n_speakers, tc_mask, frame levels, PostNet shape) must be equal, and
 *     every weight pointer NULL exactly where models[0]'s is and otherwise at the same address modulo 16; then the checks of the
 *     single-model call.
 * The workspace bounds (0 for models the call refuses) are the single-model bounds of models[0] plus the staged [2B] int32 table. */
#define FS2_MAX_VOICES 8
typedef struct fs2_acoustic_voices {
  int n;                                     /* [1, FS2_MAX_VOICES] */
  const fs2_acoustic_model* const* models;   /* host array; models[0] plans and is checked as in the single-model call */
  const fs2_acoustic_model* models_dev;      /* device copy of the n structs, read per work item */
  const int32_t* voice;                      /* [B] device */
} fs2_acoustic_voices;
size_t fs2_encode_voices_workspace_bytes(const fs2_acoustic_voices* v, int B, int L);
size_t fs2_decode_voices_workspace_bytes(const fs2_acoustic_voices* v, int B, int T);
int fs2_acoustic_encode_voices(const fs2_acoustic_voices* v, const fs2_encode_args* a, const fs2_control_args* ctl, int ragged,
                               fs2_stream_t stream);
int fs2_acoustic_decode_voices(const fs2_acoustic_voices* v, const fs2_decode_args* a, const fs2_control_args* ctl, int ragged,
                               fs2_stream_t stream);

/* ------------------------------------------------------------------ vocoder (hifigan Generator.forward) */

typedef struct fs2_vocoder_model {
  int n_mel, c0, n_stages, n_kernels, n_dil;
  int rates[FS2_MAX_STAGES], up_k[FS2_MAX_STAGES];
  int rb_k[FS2_MAX_DIL + 4]; int rb_dil[FS2_MAX_DIL + 4][FS2_MAX_DIL];
  const float *w_pre, *b_pre;                                   /* [7][n_mel][c0] */
  /* ConvTranspose1d(k = 2u) as two 2-tap phase-group convolutions writing [B][T][u*C_out]:
   *   group A: output phases p < u/2 read x[q-1], x[q];  group B: phases p >= u/2 read x[q], x[q+1]. */
  const float *w_up_a[FS2_MAX_STAGES], *w_up_b[FS2_MAX_STAGES]; /* [2][C_in][(u/2)*C_out] */
  const float *b_up[FS2_MAX_STAGES];                            /* [u*C_out] (bias tiled per phase) */
  const float *w_rb1[FS2_MAX_RESBLOCKS][FS2_MAX_DIL], *b_rb1[FS2_MAX_RESBLOCKS][FS2_MAX_DIL]; /* [k][C][C] */
  const float *w_rb2[FS2_MAX_RESBLOCKS][FS2_MAX_DIL], *b_rb2[FS2_MAX_RESBLOCKS][FS2_MAX_DIL];
  const float *w_post, *b_post;                                 /* [7][C_last], [1] */
  /* tensor-core tiles (NULL = CUDA-core kernel for that conv) */
  const float *w_pre_tc, *w_up_a_tc[FS2_MAX_STAGES], *w_up_b_tc[FS2_MAX_STAGES];
  const float *w_rb1_tc[FS2_MAX_RESBLOCKS][FS2_MAX_DIL], *w_rb2_tc[FS2_MAX_RESBLOCKS][FS2_MAX_DIL];
  int f8_mask; /* bit 0: w_pre_tc, bit 1+i: every *_tc tile of stage i is in the f16+f8 format (FS2_TC_VARIANT_F8) */
  int fused_mask; /* bit i: the ResBlock group of stage i runs on fs2_resstack, as the launches fs2_vocoder_resblock_runs plans (the
                     whole group, or runs of each ResBlock's dilations; needs f8_mask bit 1+i and a width fs2_resstack
                     serves: 8, 16, 32 or 64 channels, i.e. the last two stages of V1 and all four of V2).  In an 8-channel stage the
                     w_rb*_tc tiles are the 16 x 16 zero-padded ones fs2_resstack reads; its per-layer convs run on the exact kernel. */
  int pair_mask;  /* bit i: in stage i every (conv_k,d ; conv_k,1 ; +x) pair with k <= pair_kmax runs as one fs2_resstack launch (the
                     HBM-bound small-kernel layers: the pair's intermediate stays on chip); same requirements as fused_mask.
                     bit 8 + i: the same for a 128-channel stage i (V1's second stage), whose pairs' w_rb*_tc tiles must then be the
                     f16 + f8 tiles packed at 128 output channels per block (packing.pack_conv_tc(w, f8=True, nb=128)), not the
                     64-column blocks the per-layer conv reads; needs f8_mask bit 1+i. */
  int pair_kmax;
} fs2_vocoder_model;

/* How a stage in fused_mask cuts its ResBlock group into fs2_resstack launches (fs2_vocoder_resblock_runs).  One launch per work item
 * recomputes H halo rows on each side of its TILE output rows, so the whole group, whose H is its widest ResBlock's reach, pays for
 * that reach in every conv of every ResBlock.  The planner picks, per stage, either the whole group or, for each ResBlock j in turn,
 * consecutive runs of its dilations, each run one launch.  A run that is not the last of its ResBlock writes the fp32 residual stream
 * (alpha 1, no accumulate) that the next run reads; the last one adds alpha = 1/n_kernels times it into the stage's output as the
 * group does.  Every cut computes the same bits: each output row's sums run in the same order wherever its tile starts.  The choice
 * minimises a cost model -- MMA work on the slab rows (MT * 128 per TILE output rows) plus one fp32 write and read of every
 * intermediate -- that depends on the model only, so the offline, windowed and streams calls launch the same runs. */
typedef struct fs2_resblock_run_t {
  int32_t j;              /* kernel-size index; -1: the whole group (every kernel size, d0 = 0, d1 = n_dil) */
  int32_t d0, d1;         /* dilations [d0, d1) of ResBlock j */
  int32_t H, TILE, slab;  /* fs2_resstack_plan of the launch: halo rows per side, output rows per work item, slab rows (MT * 128) */
  double cost;            /* modelled ns per output row of the stage */
} fs2_resblock_run_t;
/* The launches of stage `stage`'s ResBlocks in issue order: writes min(count, max_runs) records to out (may be NULL) and returns the
 * count, 0 for a stage outside fused_mask, or FS2_ERR_ARG / FS2_ERR_UNSUPPORTED.  Pure host logic: no CUDA call, no pointer read. */
int fs2_vocoder_resblock_runs(const fs2_vocoder_model* m, int stage, fs2_resblock_run_t* out, int max_runs);

typedef struct fs2_vocoder_args {
  int B, T;
  const float* mel; int64_t mel_batch_stride, mel_row_stride; /* channels-last view [B][T][n_mel] */
  float* wav;                                                  /* [B][T*prod(rates)] */
  void* workspace; size_t workspace_bytes;
  /* Ragged mode: NULL (every utterance is synthesised over all T frames, as the reference does), or [B] mel-frame lengths (device,
   * clamped to [0, T]): utterance b is then synthesised exactly as a B = 1 call on its first mel_lens[b] frames, frames at or beyond
   * mel_lens[b] are never read, and wav[b, t] = 0 for t >= mel_lens[b] * prod(rates).  Every layer bounds its rows by the same array
   * (fs2_conv1d x_lens / fs2_resstack lens / fs2_conv_post lens with the layer's frames-to-rows factor as lens_scale). */
  const int32_t* mel_lens;
} fs2_vocoder_args;
/* fs2_vocoder_forward issues the launches of fs2_vocoder_window_plan(m, T, 0, T), in five workspace buffers of B * T * max(c0,
 * max_i prod(rates[0..i]) * (c0 >> (i + 1))) floats each.  A model it cannot run -- a stage with up_k != 2 * rate or an odd rate
 * (FS2_ERR_UNSUPPORTED), or a fused_mask stage without f8_mask bit 1 + i (FS2_ERR_ARG) -- is refused before any CUDA call, and
 * fs2_vocoder_workspace_bytes returns 0 for it. */
size_t fs2_vocoder_workspace_bytes(const fs2_vocoder_model* m, int B, int T);
int fs2_vocoder_forward(const fs2_vocoder_model* m, const fs2_vocoder_args* a, fs2_stream_t stream);

/* Windowed (streaming) vocoder: the waveform of the mel frames [f0, f1) of every utterance of the batch, bit for bit what
 * fs2_vocoder_forward computes there.  With up = prod(rates) and n = (min(f1, T) - f0) * up, the call writes wav[b * wav_batch_stride + i]
 * = forward's wav[b][f0 * up + i] for i < n (so wav may point at sample f0 * up of a preallocated [B][T * up] waveform, with
 * wav_batch_stride T * up, or at a [B][n] chunk); ragged mode (mel_lens) and padded mode as in fs2_vocoder_forward, so samples at or
 * past mel_lens[b] * up are zeros and an utterance that ends before f0 gives an all-zero chunk.  0 <= f0 < T and f0 < f1 (f1 may
 * exceed T), else FS2_ERR_ARG before any CUDA call.
 *   - stateless: a window depends only on mel, mel_lens, [f0, f1) and the weights; windows may be computed in any order, or twice;
 *   - every layer computes only the rows later layers need (fs2_vocoder_window_plan): a window reads the mel frames
 *     [f0 - halo, f1 + halo) of [0, mel_lens[b]) and nothing else, every intermediate likewise;
 *   - the workspace, fs2_vocoder_window_workspace_bytes(m, B, f1 - f0) or that of any wider window, does not depend on T:
 *     fs2_vocoder_window_workspace_bytes(m, B, frames) equals fs2_vocoder_streams_workspace_bytes(m, B, frames);
 *   - it issues the launches of a fs2_vocoder_forward_streams call of frames = min(f1, T) - f0 in which every stream starts at f0
 *     and has clamp(mel_lens[b], 0, T) frames (T without mel_lens): one launch stages the mel cone, then the unclipped plan of
 *     [0, frames).  Strides that are not multiples of 4 floats are FS2_ERR_UNSUPPORTED, a mel that is not 16-byte aligned FS2_ERR_ARG.
 * Every layer pads at the utterance's ends, not at the window's, and keeps the offline call's kernel choice and arithmetic per
 * output row (f8_mask, fused_mask, pair_mask, pair_kmax and the *_tc pointers apply unchanged; conv_pre runs on the backend the
 * caller's mel layout selects in fs2_vocoder_forward). */
typedef struct fs2_vocoder_window_args {
  int B, T;
  const float* mel; int64_t mel_batch_stride, mel_row_stride; /* channels-last view [B][T][n_mel], as in fs2_vocoder_args */
  float* wav;                                                  /* sample f0 * up of utterance 0; see wav_batch_stride */
  void* workspace; size_t workspace_bytes;
  const int32_t* mel_lens;                                     /* NULL or [B] mel-frame lengths (device), as in fs2_vocoder_args */
  int f0, f1;                                                  /* the window's mel frames */
  int64_t wav_batch_stride;                                    /* floats between utterances of wav (>= n) */
} fs2_vocoder_window_args;
size_t fs2_vocoder_window_workspace_bytes(const fs2_vocoder_model* m, int B, int frames);
int fs2_vocoder_forward_window(const fs2_vocoder_model* m, const fs2_vocoder_window_args* a, fs2_stream_t stream);

/* One launch of a window (fs2_vocoder_window_plan).  Rows are logical rows at the launch's rate, `scale` rows per mel frame, clipped to
 * the utterance's logical extent [0, T * scale); input and output share the rate (the ConvTranspose runs as two phase-group convs
 * whose row q holds the next rate's rows [q * u, q * u + u)).  FS2_VW_RB_GROUP is one run of fs2_vocoder_resblock_runs: j = -1 the
 * whole group, else ResBlock j's dilations [d, d1), where d1 is the next record's d if that record is a run of the same ResBlock,
 * else n_dil (the same records in the same order as fs2_vocoder_resblock_runs returns for the stage). */
enum { FS2_VW_CONV_PRE = 0, FS2_VW_UP_A = 1, FS2_VW_UP_B = 2, FS2_VW_RB_CONV1 = 3, FS2_VW_RB_CONV2 = 4, FS2_VW_RB_PAIR = 5,
       FS2_VW_RB_GROUP = 6, FS2_VW_CONV_POST = 7 };
typedef struct fs2_vocoder_window_launch_t {
  int32_t layer;        /* FS2_VW_* */
  int32_t stage, j, d;  /* upsample stage, kernel-size and dilation index (-1 where they do not apply) */
  int32_t scale;        /* rows per mel frame */
  int32_t y0, y1;       /* output rows computed */
  int32_t x0, x1;       /* input rows read */
  int32_t src;          /* launch that produced the input (the last one writing it); -1: the mel */
  int32_t res_src;      /* launch that produced the residual, read at rows [y0, y1); -1: none */
  int32_t pad_;
  double flops;         /* algorithmic FLOPs per utterance: every conv over the rows its consumers need, no tile rounding */
} fs2_vocoder_window_launch_t;
/* The launches of the window [f0, f1) of a T-frame batch in issue order, walked backward from the output samples: conv_post +-3
 * rows, a ResBlock conv (k - 1) / 2 * dilation (a fused pair or group: its total reach), a ConvTranspose phase-group pair whose output
 * rows [a, b) at the next rate read input rows [floor(a / u) - 1, ceil(b / u) + 1), conv_pre +-3.  Writes min(count, max_launches)
 * records to out (may be NULL) and returns the count, or FS2_ERR_ARG.  Pure host logic: no CUDA call.  The plan of [0, T) is
 * fs2_vocoder_forward's launch list. */
int fs2_vocoder_window_plan(const fs2_vocoder_model* m, int T, int f0, int f1, fs2_vocoder_window_launch_t* out, int max_launches);

/* Many independent streams in one call: stream b's window is its mel frames [f0[b], f0[b] + frames), each stream at its own position.
 * With up = prod(rates), wav[b * wav_batch_stride + i] = fs2_vocoder_forward(stream b alone, a B = 1 batch of n_b = mel_lens[b]
 * frames)'s wav[f0[b] * up + i] for 0 <= f0[b] * up + i < n_b * up, and 0 otherwise, for i < frames * up, bit for bit under every mask
 * and policy fs2_vocoder_forward_window honours.  A stream's output does not depend on the other streams of the call.
 *   - the host never reads f0, mel_lens or the pointer table: the launch plan is the unclipped plan of [0, frames)
 *     (fs2_vocoder_window_plan's rows of a window that no utterance end clips), the grid is sized from B and that plan, and each
 *     kernel bounds utterance b by its own origin: row r of a layer with `scale` rows per frame is live iff
 *     0 <= r + f0[b] * scale < n_b * scale;
 *   - any device values are memory-safe: stream b's mel is read only at rows of [0, n_b) inside its window's cone; f0[b] >= n_b or
 *     n_b <= 0 gives an all-zero chunk, and rows before a negative f0[b] read as zero;
 *   - one launch stages every stream's mel cone ([B][cone rows][n_mel]), f0 and mel_lens into the workspace; the rest are the
 *     launches of the unclipped plan of [0, frames);
 *   - B <= 0, frames <= 0, a NULL pointer, wav_batch_stride < frames * up with B > 1, or a workspace below
 *     fs2_vocoder_streams_workspace_bytes(m, B, frames) is FS2_ERR_ARG before any CUDA call.  That bound depends on B and frames only:
 *     the plan's five buffers, the staged mel cone and two [B] int32 tables. */
typedef struct fs2_vocoder_streams_args {
  int B, frames;                  /* B streams, `frames` mel frames each */
  const float* const* mel;        /* [B] device array: stream b's mel rows, n_mel contiguous floats per row, 16-byte aligned */
  const int32_t* mel_lens;        /* [B] device: stream b's total frames n_b */
  const int32_t* f0;              /* [B] device: stream b's first frame in this call */
  float* wav; int64_t wav_batch_stride;   /* [B][frames * up] */
  void* workspace; size_t workspace_bytes;
} fs2_vocoder_streams_args;
size_t fs2_vocoder_streams_workspace_bytes(const fs2_vocoder_model* m, int B, int frames);
int fs2_vocoder_forward_streams(const fs2_vocoder_model* m, const fs2_vocoder_streams_args* a, fs2_stream_t stream);

/* Streams whose mel is a ring: fs2_vocoder_forward_streams, but stream b's frame t lives at row t mod cap[b] of its cap[b]-row buffer
 * mel[b] (n_mel contiguous floats per row, 16-byte aligned).  With n_b = mel_lens[b], the output equals fs2_vocoder_forward_streams on
 * the stream's unwrapped frames bit for bit, provided every frame of the window's cone inside [0, n_b) is still in the ring (within the
 * last cap[b] frames written).  A finished mel is the ring cap[b] = n_b, which never wraps.
 *   - the host never reads cap: the row index is reduced mod cap[b] on the device, so the reads stay inside the cap[b] rows at
 *     mel[b]; cap[b] <= 0 gives an all-zero chunk;
 *   - the launches, workspace bound (fs2_vocoder_streams_workspace_bytes) and argument checks are those of
 *     fs2_vocoder_forward_streams, plus FS2_ERR_ARG for a NULL cap. */
typedef struct fs2_vocoder_streams_ring_args {
  int B, frames;
  const float* const* mel;        /* [B] device array: stream b's ring of cap[b] rows */
  const int32_t* mel_lens;        /* [B] device: frames of stream b that exist (written so far, or its total) */
  const int32_t* f0;              /* [B] device: stream b's first frame in this call */
  float* wav; int64_t wav_batch_stride;
  void* workspace; size_t workspace_bytes;
  const int32_t* cap;             /* [B] device: ring rows of stream b */
} fs2_vocoder_streams_ring_args;
int fs2_vocoder_forward_streams_ring(const fs2_vocoder_model* m, const fs2_vocoder_streams_ring_args* a, fs2_stream_t stream);

/* Streams of several generators in one call: fs2_vocoder_forward_streams_ring (cap may be NULL: no rings, as
 * fs2_vocoder_forward_streams), but stream b is vocoded with generator gen[b] of models[0 .. n_models): its output equals that call with
 * models[gen[b]] alone bit for bit, whatever the other streams' generators.  The generators share one architecture and weight format
 * (fine-tuned copies of one checkpoint, or V1 checkpoints trained apart), so the call plans once, on models[0]: its launches, grid and
 * launch count are those of fs2_vocoder_forward_streams at the same B and frames, and every work item reads its own stream's weights.
 *   - models_dev: a device copy of the n_models structs models points at (the pointers inside are device pointers anyway); the kernels
 *     read each weight's pointer from models_dev[gen[b]], so it must stay equal to the host array while the call runs;
 *   - the host never reads gen: the staging launch clamps it with the origin and length tables, and a stream whose gen[b] lies outside
 *     [0, n_models) gets an all-zero chunk (as cap[b] <= 0 does) without changing the other streams;
 *   - FS2_ERR_ARG before any CUDA call for n_models outside [1, FS2_MAX_GENERATORS], a NULL model, gen or models_dev, and a model whose
 *     architecture (n_mel, c0, stages, rates, up_k, ResBlock kernels and dilations), masks (f8_mask, fused_mask, pair_mask, pair_kmax) or
 *     weight format differs from models[0]'s -- every weight pointer must be NULL where models[0]'s is (which *_tc tiles exist, and so
 *     which convs, conv_pre included, take the tensor cores) and otherwise lie at the same address modulo 16; then the checks of
 *     fs2_vocoder_forward_streams.  The workspace bound, fs2_vocoder_streams_multi_workspace_bytes (0 for models the call refuses), is
 *     fs2_vocoder_streams_workspace_bytes of models[0] plus the staged generator table. */
#define FS2_MAX_GENERATORS 8
typedef struct fs2_vocoder_streams_multi_args {
  int B, frames;
  const float* const* mel;        /* [B] device array: stream b's mel rows (its ring of cap[b] rows when cap is set) */
  const int32_t* mel_lens;        /* [B] device */
  const int32_t* f0;              /* [B] device */
  float* wav; int64_t wav_batch_stride;
  void* workspace; size_t workspace_bytes;
  const int32_t* cap;             /* [B] device, or NULL */
  const int32_t* gen;             /* [B] device: stream b's generator index */
  const fs2_vocoder_model* models_dev;   /* [n_models] device copy of the models' structs */
} fs2_vocoder_streams_multi_args;
size_t fs2_vocoder_streams_multi_workspace_bytes(const fs2_vocoder_model* const* models, int n_models, int B, int frames);
int fs2_vocoder_forward_streams_multi(const fs2_vocoder_model* const* models, int n_models, const fs2_vocoder_streams_multi_args* a,
                                      fs2_stream_t stream);

/* Appending arriving mel frames to rings, every stream's in one launch: record r copies `count` frames, source frame src_frame + i at
 * src + (src_frame + i) * frame_stride + c * channel_stride (floats) for channel c, to ring row (dst_frame + i) mod cap of `ring`
 * ([cap][n_mel] channels-last, 16-byte aligned), for i < count.  Any strides: FastSpeech2's postnet_mel[b] is frame_stride n_mel,
 * channel_stride 1 (float4 loads when aligned), an [n_mel, m] channel-major block frame_stride 1, channel_stride m (transposed on the
 * way in).  Every ring row is written with float4 stores.
 *   - the host never reads the table: the grid is sized from n_records and max_count, count is clamped to [0, max_count], and a count
 *     past cap copies only its last cap frames (what copying in order would leave); a record with cap <= 0 or a ring that is not
 *     16-byte aligned writes nothing;
 *   - a NULL table, n_records <= 0 or max_count <= 0 is FS2_ERR_ARG, n_mel not a positive multiple of 4 FS2_ERR_UNSUPPORTED, before any
 *     CUDA call.  Records of one launch must not write the same ring rows. */
typedef struct fs2_mel_ring_record_t {
  const float* src;
  int64_t frame_stride, channel_stride, src_frame;
  float* ring;
  int64_t dst_frame;
  int32_t cap, count;
} fs2_mel_ring_record_t;
typedef struct fs2_mel_ring_append_args {
  const fs2_mel_ring_record_t* table;   /* [n_records] device */
  int n_records, n_mel, max_count;
} fs2_mel_ring_append_args;
int fs2_mel_ring_append(const fs2_mel_ring_append_args* a, fs2_stream_t stream);

/* ------------------------------------------------------------------ sample-rate conversion of the waveform (scipy.signal.resample_poly)
 *
 * up / down is fs_out / fs_in reduced, max(up, down) <= FS2_RESAMPLE_MAX_FACTOR.  With half_len = 10 * max(up, down) and the
 * (2 half_len + 1)-tap Kaiser(5.0) low-pass h that resample_poly designs (firwin(...) * up), output j of a row of n input samples is
 *     y[j] = sum over ascending i of x[i] * h[j * down - i * up + half_len],  0 <= i < n,  0 <= j * down - i * up + half_len <= 2 half_len,
 * for j < n_out = ceil(n * up / down), and 0 for j >= n_out (zero padding: inputs outside [0, n) are zero).  The sum runs in fp32, one
 * fmaf per tap in descending tap order (ascending i), from fp32 taps, so an output's bits depend on its inputs only, never on where a
 * window or chunk boundary falls.  Output j reads the K contiguous inputs [q - K + 1, q], q = floor((j * down + half_len) / up), with the
 * taps of phase p = (j * down + half_len) mod up.
 * taps: [up][K] fp32, taps[p * K + k] = h[p + k * up], zero where p + k * up > 2 half_len; K = ceil((2 half_len + 1) / up).
 * pcm16 != 0 writes int16 (trunc(y * scale) clamped to [-32768, 32767], as fs2_wav_to_int16; resampled audio can ring past +-1, so the
 * clamp is reachable here) instead of fp32.
 * Every call returns FS2_ERR_ARG before any CUDA call for a ratio, K or pointer that breaks these rules, and FS2_ERR_UNSUPPORTED when the
 * tap table does not fit the device's shared memory (it always fits an H100's for max(up, down) <= FS2_RESAMPLE_MAX_FACTOR). */
#define FS2_RESAMPLE_MAX_FACTOR 2048

/* Offline: every row of x [B][N] (batch stride in floats), row b over its own min(lens[b] * lens_scale, N) samples when lens is set
 * (device int32, clamped, never read by the host), so that row b equals a B = 1 call on its first lens[b] * lens_scale samples and its
 * outputs at or past ceil(lens[b] * lens_scale * up / down) are zeros.  y: [B][ceil(N * up / down)] with batch stride y_batch_stride
 * (elements of fp32 or int16). */
typedef struct fs2_resample_args {
  int B, up, down, K;
  const float* taps;
  const float* x; int64_t x_batch_stride, N;
  const int32_t* lens; int32_t lens_scale;
  void* y; int64_t y_batch_stride;
  int32_t pcm16; float scale;
} fs2_resample_args;
int fs2_resample(const fs2_resample_args* a, fs2_stream_t stream);

/* Window: outputs [j0, j1) of every row (0 <= j0 < j1 <= ceil(N * up / down)), written to y[b * y_batch_stride + j - j0], from input
 * samples [i0, i2) given in two pieces: x0 holds samples [i0, i1) (x0[b * x0_batch_stride + i - i0]), x1 holds [i1, i2) (may be NULL
 * when i1 == i2) -- typically the previous chunk's tail and the current chunk.  N and lens bound the rows as in fs2_resample.  Every
 * input of [0, N) the outputs read must lie in [i0, i2), else FS2_ERR_ARG (pure integer host check); inputs at or past a row's
 * lens[b] * lens_scale are zeros whether given or not.  The outputs equal fs2_resample's bit for bit. */
typedef struct fs2_resample_window_args {
  int B, up, down, K;
  const float* taps;
  const float* x0; int64_t x0_batch_stride;
  const float* x1; int64_t x1_batch_stride;
  int64_t i0, i1, i2, N;
  const int32_t* lens; int32_t lens_scale;
  int64_t j0, j1;
  void* y; int64_t y_batch_stride;
  int32_t pcm16; float scale;
} fs2_resample_window_args;
int fs2_resample_window(const fs2_resample_window_args* a, fs2_stream_t stream);

/* Streams: one device record per stream, each stream at its own position, in one launch (the resampling step of a stream pool).  Stream b
 * writes its outputs [j0, j1) to y[b * y_batch_stride + j - j0] from its pieces x0 = samples [i0, i1) and x1 = samples [i1, i2) of a
 * stream of n input samples, equal bit for bit to fs2_resample of that stream alone.  The host never reads the table: the grid is
 * sized from max_out, j1 - j0 is clamped to [0, max_out], and an input of [0, n) outside [i0, i2) reads as zero (the caller provides
 * every input its outputs need; Python's stream_pool does by construction). */
typedef struct fs2_resample_stream_t {
  const float *x0, *x1;
  int64_t i0, i1, i2, n, j0, j1;
} fs2_resample_stream_t;
typedef struct fs2_resample_streams_args {
  int B, up, down, K;
  const float* taps;
  const fs2_resample_stream_t* table;   /* [B] device */
  int64_t max_out;
  void* y; int64_t y_batch_stride;
  int32_t pcm16; float scale;
} fs2_resample_streams_args;
int fs2_resample_streams(const fs2_resample_streams_args* a, fs2_stream_t stream);

/* Mixed streams: as fs2_resample_streams, but each stream names its own filter in a table of n_filters (1..FS2_RESAMPLE_MAX_FILTERS)
 * filters passed by value, and its own output encoding, so that streams at different rates and sample types share one launch.
 * Encodings: FS2_RESAMPLE_F32 writes fp32; FS2_RESAMPLE_PCM16 int16 as pcm16 above; FS2_RESAMPLE_ULAW / FS2_RESAMPLE_ALAW one byte,
 * the ITU-T G.711 mu-law / A-law code of that int16 sample (equal to Python's audioop.lin2ulaw / lin2alaw on 16-bit input).
 * A filter is a ratio with its taps as above, or the identity: up == down == 1, K == 1 and taps a one-tap table of 1.0f, whose output
 * j is input j (with PCM16, fs2_wav_to_int16's bits; with F32, x + 0.0f, so -0.0f becomes +0.0f).  The identity is accepted here only.
 * Stream b writes outputs [j0, j1) (j1 - j0 clamped to [0, max_out]) to the bytes at y + y_offset, elements of its encoding.  The host
 * never reads the table; a record whose filter is outside [0, n_filters), whose encoding is unknown, or whose y_offset is negative or
 * not a multiple of 16 writes nothing.  The host refuses before any CUDA call (FS2_ERR_ARG) a bad B, n_filters, ratio, K or taps, a
 * NULL table, max_out < 1, and a y that is NULL or not 16-byte aligned.  Dynamic shared memory is the largest of the filters' needs. */
#define FS2_RESAMPLE_MAX_FILTERS 8
#define FS2_RESAMPLE_F32 0
#define FS2_RESAMPLE_PCM16 1
#define FS2_RESAMPLE_ULAW 2
#define FS2_RESAMPLE_ALAW 3
typedef struct fs2_resample_filter_t {
  int32_t up, down, K;
  const float* taps;                    /* [up][K] device */
} fs2_resample_filter_t;
typedef struct fs2_resample_mixed_stream_t {
  const float *x0, *x1;
  int64_t i0, i1, i2, n, j0, j1;        /* as fs2_resample_stream_t */
  int32_t filter, encoding;
  int64_t y_offset;                     /* bytes from y */
} fs2_resample_mixed_stream_t;
typedef struct fs2_resample_mixed_args {
  int B, n_filters;
  fs2_resample_filter_t filters[FS2_RESAMPLE_MAX_FILTERS];
  const fs2_resample_mixed_stream_t* table;   /* [B] device */
  int64_t max_out;
  void* y;
  float scale;
} fs2_resample_mixed_args;
int fs2_resample_streams_mixed(const fs2_resample_mixed_args* a, fs2_stream_t stream);

/* ------------------------------------------------------------------ misc */
int fs2_abi_version(void);                 /* bumps when any struct above changes */
int64_t fs2_kernel_launch_count(void);     /* kernels launched by this library since load (process-wide) */
const char* fs2_build_info(void);          /* "sm_90a ..." */
/* sizeof of a struct above (binding self-check), fs2_<name>[_args]: 0 conv1d, 1 layernorm, 2 attention, 3 embed, 4 rowbias,
 * 5 variance_head, 6 durations, 7 length_regulate, 8 conv_post, 9 acoustic_model, 10 encode, 11 decode, 12 vocoder_model,
 * 13 vocoder, 14 resstack, 15 wav_int16, 16 conv_tc_plan_t, 17 conv_simt_plan_t, 18 resstack_plan_t.  Like fs2_control_args,
 * fs2_vocoder_window_args (80 bytes), fs2_vocoder_window_launch_t (56 bytes), fs2_vocoder_streams_args (64 bytes) and the resampler's
 * structs (fs2_resample_args 88, fs2_resample_window_args 144, fs2_resample_stream_t 64, fs2_resample_streams_args 64 bytes; added at
 * ABI 12 without a bump, since no existing struct changed; then fs2_resample_filter_t 24, fs2_resample_mixed_stream_t 80 and
 * fs2_resample_mixed_args 232 bytes, likewise; then fs2_vocoder_streams_ring_args 72, fs2_mel_ring_record_t 56 and
 * fs2_mel_ring_append_args 24 bytes, likewise; then fs2_vocoder_streams_multi_args 88 bytes, likewise; then fs2_acoustic_voices 32 bytes,
 * likewise) are not in the table: the binding pins their sizes. */
size_t fs2_struct_size(int which);
/* Re-entrancy: the library keeps no mutable process-wide state behind these calls except (a) a per-device table of one-time
 * cudaFuncSetAttribute opt-ins and SM counts, filled under a mutex for the device that is CURRENT when a call is made -- make the
 * device that owns the stream current before calling -- (b) the launch counter above and (c) the profiling state below, which is
 * per host thread.
 * Per-kernel-class device timing for bench.py's roofline (CUDA events recorded around each launch on the launch stream).
 * Classes: 0 tensor-core kernels (conv1d implicit GEMM + fused ResBlock group), 1 attention, 2 layernorm, 3 everything else, 4 fp32 CUDA-core conv1d.  begin() arms it, end() synchronises the
 * recorded events, fills ms/flops/launches per class (arrays of FS2_PROF_CLASSES) and disarms.  Not for timed regions. */
#define FS2_PROF_CLASSES 5
int fs2_profile_begin(void);
int fs2_profile_end(double* ms, double* flops, int64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* FS2B200_H */
