// Host-side orchestration of the two forward passes and the extern "C" surface declared in include/fs2b200.h.
// No allocation, no synchronisation: every launch goes to the caller's stream, temporaries come from the caller's workspace.
#include <mutex>
#include <new>
#include <vector>

#include "common.cuh"

namespace fs2 {

std::atomic<unsigned long long> g_launch_count{0};

// ------------------------------------------------------------------ per-device setup state
static DevState g_dev[FS2_MAX_DEVICES];
static std::mutex g_dev_mutex;
DevState* dev_state(int* err) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess || dev < 0 || dev >= FS2_MAX_DEVICES) {
    if (err) *err = e != cudaSuccess ? FS2_ERR_CUDA - (int)e : FS2_ERR_UNSUPPORTED;
    return nullptr;
  }
  DevState* d = &g_dev[dev];
  if (d->num_sms.load(std::memory_order_acquire) == 0) {
    int n = 0;
    e = cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess || n <= 0) {
      if (err) *err = FS2_ERR_CUDA - (int)e;
      return nullptr;
    }
    d->num_sms.store(n, std::memory_order_release);
  }
  return d;
}
int dev_once(std::atomic<bool>& ready, cudaError_t (*setup)()) {
  if (ready.load(std::memory_order_acquire)) return FS2_OK;
  std::lock_guard<std::mutex> lock(g_dev_mutex);
  if (ready.load(std::memory_order_relaxed)) return FS2_OK;
  const cudaError_t e = setup();
  if (e != cudaSuccess) return FS2_ERR_CUDA - (int)e;
  ready.store(true, std::memory_order_release);
  return FS2_OK;
}

// ------------------------------------------------------------------ per-launch profiling (off unless armed; state is per host thread)
thread_local bool g_prof_on = false;
struct ProfRec { cudaEvent_t a, b; int cls; double flops; };
static thread_local std::vector<ProfRec> g_prof;
static thread_local cudaEvent_t g_prof_pending;
void prof_before(cudaStream_t s) {
  if (!g_prof_on) return;
  cudaEventCreate(&g_prof_pending);
  cudaEventRecord(g_prof_pending, s);
}
void prof_after(cudaStream_t s, int cls, double flops) {
  if (!g_prof_on) return;
  ProfRec r;
  r.a = g_prof_pending; r.cls = cls; r.flops = flops;
  cudaEventCreate(&r.b);
  cudaEventRecord(r.b, s);
  g_prof.push_back(r);
}

// kernels / launchers defined in the other translation units
int conv1d_simt(const fs2_conv1d_args* a, cudaStream_t s);
int conv1d_tc(const fs2_conv1d_args* a, cudaStream_t s);
int attention_fused(const fs2_attention_args* a, void* ws, size_t ws_bytes, cudaStream_t s, bool ragged = false);
size_t attention_fused_workspace(int B, int T, int H);
bool conv_tc_supported(const fs2_conv1d_args* a);
int conv_tc_nb(int N, int nb_max);
int conv_tc_plan_query(const fs2_conv1d_args* a, int num_sms, int* out);

// backend dispatch of the fs2_conv1d contract
static int conv1d_dispatch(const fs2_conv1d_args* a, cudaStream_t s) {
  if (!a) return FS2_ERR_ARG;
  if (a->x_lens && a->lens_scale < 1) return FS2_ERR_ARG;
  if (a->backend == FS2_CONV_TC) return conv1d_tc(a, s);
  if (a->backend == FS2_CONV_AUTO && a->w_tc && conv_tc_supported(a)) return conv1d_tc(a, s);
  return conv1d_simt(a, s);
}
int attention_simt(const fs2_attention_args* a, cudaStream_t s, bool ragged = false, int fused_from = 0);
int embed_positions(const fs2_embed_args* a, cudaStream_t s);
int add_speaker(const fs2_rowbias_args* a, cudaStream_t s);
int layernorm(const fs2_layernorm_args* a, cudaStream_t s);
int variance_head(const fs2_variance_head_args* a, cudaStream_t s);
int durations(const fs2_durations_args* a, cudaStream_t s, const int32_t* src_lens = nullptr);
int length_regulate(const fs2_length_regulate_args* a, cudaStream_t s);
int conv_post(const fs2_conv_post_args* a, cudaStream_t s);
int resstack(const fs2_resstack_args* a, cudaStream_t s);
int wav_to_int16(const fs2_wav_int16_args* a, cudaStream_t s);
int resstack_plan(const fs2_resstack_args* a, int num_sms, int* out);
int transpose_bct_to_btc(const float* in, float* out, int B, int C, int T, cudaStream_t s);
int add_positions(float* x, const float* pos, int B, int T, int D, cudaStream_t s);
int zero_tail(float* y0, float* y1, const int32_t* lens, int B, int T, int C, cudaStream_t s);

// ------------------------------------------------------------------ workspace bump allocator
struct Arena {
  char* base; size_t cap, off;
  bool dry;  // dry run: only measure
  explicit Arena(void* p, size_t n) : base((char*)p), cap(n), off(0), dry(p == nullptr) {}
  float* f32(size_t n) { return (float*)take(n * sizeof(float)); }
  void* take(size_t bytes) {
    const size_t a = (off + 255) & ~(size_t)255;
    off = a + bytes;
    if (dry) return (void*)(uintptr_t)256;  // non-null dummy
    if (off > cap) return nullptr;
    return base + a;
  }
};

// fs2_conv1d arguments for contiguous [B][T][Cin] input, [B][T][N] output and residual, `taps` with "same" padding at dilation 1.
// The rest starts at its identity: bias and residual off, alpha 1, no activations, FS2_CONV_AUTO, no row_lens / x_lens.
// Call sites set the weights and whatever else differs by field name.
static fs2_conv1d_args conv_args(const float* x, int B, int T, int Cin, int N, int taps, float* y) {
  fs2_conv1d_args a{};
  a.x = x; a.x_batch_stride = (int64_t)T * Cin; a.x_row_stride = Cin;
  a.B = B; a.T = T; a.Cin = Cin;
  a.N = N; a.taps = taps; a.dilation = 1; a.pad_left = (taps - 1) / 2;
  a.backend = FS2_CONV_AUTO; a.alpha = 1.f;
  a.res_batch_stride = (int64_t)T * N; a.res_row_stride = N;
  a.y = y; a.y_batch_stride = (int64_t)T * N; a.y_row_stride = N;
  a.lens_scale = 1;
  return a;
}

// How the convs of one FFT block, variance predictor or the decoder's mel_linear + PostNet run, decided once per block.
//  EXACT:     fp32 CUDA-core kernel (w_tc is not passed).
//  TC:        split-precision tensor-core kernel with variant `tcv` wherever conv1d_dispatch supports the shape.
//  SEGMENTED: K-segmented tensor-core convolution for the layers that feed the discrete decisions (encoder, predictors): the sum over
//             taps and input channels is cut into (tap, 256-channel) slices; each slice is one work unit of 16 K-steps with separate
//             accumulators for the hi*hi term and the cross terms (FS2_TC_VARIANT_NB64 | FS2_TC_VARIANT_SEGMENTED, one launch per
//             conv), and the slices are added in fp32 round-to-nearest by the epilogue's accumulate path.  That bounds the tensor
//             core's truncating accumulation to 16 steps per chain (a single k = 9 launch has 432) and brings the error back to the
//             fp32 CUDA-core kernel's level (scripts/flip_census.py).  w_tc: taps * (Cin/256) tile buffers of 128 + 1024*N bytes
//             (packing.pack_conv_tc_segments).  No output activation: a following ReLU is applied by the consumer (in_act of the
//             next conv / pre_relu of the LayerNorm).
struct ConvMode {
  enum { EXACT, TC, SEGMENTED } path;
  unsigned tcv;
  void weights(fs2_conv1d_args& a, const float* w, const float* w_tc, const float* bias) const {
    a.bias = bias;
    if (path == SEGMENTED) {
      a.w = nullptr; a.w_tc = w_tc; a.backend = FS2_CONV_TC; a.tc_variant = FS2_TC_VARIANT_NB64 | FS2_TC_VARIANT_SEGMENTED;
    } else {
      a.w = w; a.w_tc = path == TC ? w_tc : nullptr; a.tc_variant = tcv;
    }
  }
};

struct FftBufs { float *x, *tmp, *qkv, *ctx, *hid; void* att_ws; size_t att_bytes; };

// Ragged mode (fs2_acoustic_encode_ragged / fs2_acoustic_decode_ragged): utterance b is bounded by lens[b] rows in every layer, so it is
// computed exactly as a B = 1 call on those rows would compute it.  Each conv gets the lengths as x_lens (lens_scale 1): it reads rows
// at or beyond lens[b] as zero and leaves its output rows there unspecified; the LayerNorms zero them.  `rag` is that x_lens, or NULL.
static const int32_t* ragged_lens(bool ragged, const int32_t* lens) { return ragged ? lens : nullptr; }

// One FFT block in place on bufs.x  (transformer/Layers.py:21-30)
static int fft_block(cudaStream_t s, const fs2_acoustic_model* m, const fs2_fft_block_weights& w, const FftBufs& f, int B, int T,
                     const int32_t* lens, ConvMode mode, bool ragged) {
  const int D = m->d_model, F = m->d_inner;
  const bool seg = mode.path == ConvMode::SEGMENTED;
  const int32_t* rag = ragged_lens(ragged, lens);
  if (seg && (!w.w_qkv_tc || !w.w_o_tc || !w.w_1_tc || !w.w_2_tc || m->k2 != 1)) return FS2_ERR_ARG;
  fs2_conv1d_args c = conv_args(f.x, B, T, D, 3 * D, 1, f.qkv);
  mode.weights(c, w.w_qkv, w.w_qkv_tc, w.b_qkv);
  c.x_lens = rag;
  FS2_TRY(conv1d_dispatch(&c, s));
  fs2_attention_args at{};
  at.qkv = f.qkv; at.ctx = f.ctx; at.B = B; at.T = T; at.H = m->n_head; at.Dh = D / m->n_head; at.key_lens = lens;
  at.scale = 1.0f / sqrtf((float)(D / m->n_head));
  if (mode.path == ConvMode::TC && f.att_ws && T >= 128) {           // one fused tensor-core kernel: S stays in registers, any length
    FS2_TRY(attention_fused(&at, f.att_ws, f.att_bytes, s, ragged));
    // ragged: the fused kernel takes the utterances of >= 128 rows, the exact kernel the shorter ones -- the backends a B = 1 call picks
    if (ragged) FS2_TRY(attention_simt(&at, s, true, 128));
  } else {
    FS2_TRY(attention_simt(&at, s, ragged, 0));
  }
  c = conv_args(f.ctx, B, T, D, D, 1, f.tmp);
  mode.weights(c, w.w_o, w.w_o_tc, w.b_o);
  c.res = f.x;
  c.x_lens = rag;
  FS2_TRY(conv1d_dispatch(&c, s));
  fs2_layernorm_args n{};                                           // both LayerNorms: tmp -> x, padded rows zeroed
  n.x = f.tmp; n.y = f.x; n.B = B; n.T = T; n.C = D; n.eps = 1e-5f; n.row_lens = lens;
  n.gamma = w.ln1_g; n.beta = w.ln1_b;
  FS2_TRY(layernorm(&n, s));
  // conv-FFN.  K-segmented: w_1 leaves the pre-activation hidden and the ReLU is w_2's input activation (leaky_relu with slope 0)
  c = conv_args(f.x, B, T, D, F, m->k1, f.hid);
  mode.weights(c, w.w_1, w.w_1_tc, w.b_1);
  if (!seg) c.out_act = FS2_ACT_RELU;
  c.x_lens = rag;
  FS2_TRY(conv1d_dispatch(&c, s));
  c = conv_args(f.hid, B, T, F, D, m->k2, f.tmp);
  mode.weights(c, w.w_2, w.w_2_tc, w.b_2);
  c.res = f.x;
  if (seg) { c.in_act = FS2_ACT_LRELU; c.in_slope = 0.f; }
  c.x_lens = rag;
  FS2_TRY(conv1d_dispatch(&c, s));
  n.gamma = w.ln2_g; n.beta = w.ln2_b;
  return layernorm(&n, s);
}

static bool model_ok(const fs2_acoustic_model* m) {
  return m && m->d_model > 0 && m->n_head > 0 && m->d_model % m->n_head == 0 && m->n_enc >= 0 && m->n_enc <= FS2_MAX_LAYERS &&
         m->n_dec >= 0 && m->n_dec <= FS2_MAX_LAYERS && m->n_postnet >= 0 && m->n_postnet <= FS2_MAX_POSTNET && m->d_inner > 0 &&
         m->n_mel > 0 && m->vp_filter > 0;
}

static FftBufs fft_bufs(Arena& ar, const fs2_acoustic_model* m, size_t rows, int B = 0, int T = 0, bool tc_attention = false) {
  FftBufs f;
  f.att_ws = nullptr; f.att_bytes = 0;
  if (tc_attention && T >= 128) {
    f.att_bytes = attention_fused_workspace(B, T, m->n_head);
    f.att_ws = ar.take(f.att_bytes);
  }
  f.x = ar.f32(rows * m->d_model);
  f.tmp = ar.f32(rows * m->d_model);
  f.qkv = ar.f32(rows * 3 * m->d_model);
  f.ctx = ar.f32(rows * m->d_model);
  f.hid = ar.f32(rows * m->d_inner);
  return f;
}

// VariancePredictor.forward (+ bucketize / embedding add when bins != NULL) on rows [B][T]  (model/modules.py:242-250, :80-100).
// `head` carries the caller's part of the head's arguments: B, L = T, lens, control, target, bins, emb, pred_out, and x, which is
// both the predictor's input and where the embedding is added.  Ragged: the convs and LayerNorms are bounded by head.lens.
static int run_predictor(cudaStream_t s, const fs2_acoustic_model* m, const fs2_predictor_weights& w, fs2_variance_head_args head,
                         float* h1, float* h2, bool ragged) {
  const int B = head.B, T = head.L, k = m->vp_kernel, D = m->d_model, VF = m->vp_filter;
  const bool seg = (m->tc_mask & FS2_TC_PREDICTORS) && w.w_c1_tc && w.w_c2_tc;   // K-segmented: the ReLU is applied by the LayerNorm
  const ConvMode mode{seg ? ConvMode::SEGMENTED : ConvMode::EXACT, 0};
  const int32_t* rag = ragged_lens(ragged, head.lens);
  fs2_layernorm_args n{};                                           // both LayerNorms: h1 -> h2, unmasked (ragged: masked)
  n.x = h1; n.y = h2; n.B = B; n.T = T; n.C = VF; n.eps = 1e-5f; n.pre_relu = seg; n.row_lens = rag;
  fs2_conv1d_args c = conv_args(head.x, B, T, D, VF, k, h1);
  mode.weights(c, w.w_c1, w.w_c1_tc, w.b_c1);
  if (!seg) c.out_act = FS2_ACT_RELU;
  c.x_lens = rag;
  FS2_TRY(conv1d_dispatch(&c, s));
  n.gamma = w.ln1_g; n.beta = w.ln1_b;
  FS2_TRY(layernorm(&n, s));
  c = conv_args(h2, B, T, VF, VF, k, h1);
  mode.weights(c, w.w_c2, w.w_c2_tc, w.b_c2);
  c.pad_left = 1;                                                   // padding=1 is hard-coded upstream
  if (!seg) c.out_act = FS2_ACT_RELU;
  c.x_lens = rag;
  FS2_TRY(conv1d_dispatch(&c, s));
  n.gamma = w.ln2_g; n.beta = w.ln2_b;
  FS2_TRY(layernorm(&n, s));
  head.h = h2; head.w = w.w_out; head.b = w.b_out; head.C = VF; head.n_edges = m->n_bins - 1; head.D = D;
  return variance_head(&head, s);
}

// ------------------------------------------------------------------ phase 1
// ragged: utterance b has src_lens[b] phonemes; x_adapted rows at or beyond it are left unspecified.
static int encode_impl(const fs2_acoustic_model* m, const fs2_encode_args* a, cudaStream_t s, Arena& ar, bool ragged) {
  const int B = a->B, L = a->L, D = m->d_model, VF = m->vp_filter;
  const size_t rows = (size_t)B * L;
  FftBufs f = fft_bufs(ar, m, rows);
  float* h1 = ar.f32(rows * VF);
  float* h2 = ar.f32(rows * VF);
  if (ar.dry) return FS2_OK;
  if (!f.x || !f.tmp || !f.qkv || !f.ctx || !f.hid || !h1 || !h2) return FS2_ERR_WORKSPACE;
  if (L > m->enc_pos_rows) return FS2_ERR_ARG;

  fs2_embed_args e{};
  e.ids = a->texts; e.table = m->word_emb; e.pos = m->enc_pos; e.y = f.x; e.B = B; e.L = L; e.D = D; e.n_vocab = m->n_vocab;
  FS2_TRY(embed_positions(&e, s));
  const ConvMode enc_mode{(m->tc_mask & FS2_TC_ENCODER) ? ConvMode::SEGMENTED : ConvMode::EXACT, 0};   // exact attention either way
  for (int i = 0; i < m->n_enc; i++) FS2_TRY(fft_block(s, m, m->enc[i], f, B, L, a->src_lens, enc_mode, ragged));
  if (m->spk_emb) {
    if (!a->speakers) return FS2_ERR_ARG;
    fs2_rowbias_args r{};
    r.x = f.x; r.table = m->spk_emb; r.idx = a->speakers; r.B = B; r.L = L; r.D = D; r.n_rows = m->n_speakers;
    FS2_TRY(add_speaker(&r, s));
  }
  // x_adapted starts as the encoder output; pitch / energy embeddings are added in place (modules.py:117-126)
  cudaError_t ce = cudaMemcpyAsync(a->x_adapted, f.x, rows * D * sizeof(float), cudaMemcpyDeviceToDevice, s);
  if (ce != cudaSuccess) return FS2_ERR_CUDA - (int)ce;

  // duration on the un-embedded x; pitch on x; energy on x + pitch embedding.  energy uses p_control (modules.py:124).
  fs2_variance_head_args v{};
  v.x = a->x_adapted; v.B = B; v.L = L; v.lens = a->src_lens; v.control = 1.f; v.pred_out = a->logd_pred;
  FS2_TRY(run_predictor(s, m, m->dur, v, h1, h2, ragged));
  v.control = a->p_control;
  if (!m->pitch_frame_level) {
    if (!a->p_pred) return FS2_ERR_ARG;
    v.target = a->p_target; v.bins = m->pitch_bins; v.emb = m->pitch_emb; v.pred_out = a->p_pred;
    FS2_TRY(run_predictor(s, m, m->pitch, v, h1, h2, ragged));
  }
  if (!m->energy_frame_level) {
    if (!a->e_pred) return FS2_ERR_ARG;
    v.target = a->e_target; v.bins = m->energy_bins; v.emb = m->energy_emb; v.pred_out = a->e_pred;
    FS2_TRY(run_predictor(s, m, m->energy, v, h1, h2, ragged));
  }

  fs2_durations_args d{};
  d.src = a->d_target ? a->d_target : a->logd_pred; d.use_target = a->d_target != nullptr; d.d_control = a->d_control;
  d.B = B; d.L = L; d.d_rounded = a->d_target ? nullptr : a->d_rounded; d.cum = a->cum_dur; d.mel_lens = a->mel_lens;
  d.mel_lens32 = a->mel_lens32; d.len_stats = a->len_stats;
  FS2_TRY(durations(&d, s, ragged_lens(ragged, a->src_lens)));
  if (a->len_stats_host) {
    ce = cudaMemcpyAsync(a->len_stats_host, a->len_stats, 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
    if (ce != cudaSuccess) return FS2_ERR_CUDA - (int)ce;
  }
  return FS2_OK;
}

// ------------------------------------------------------------------ phase 2
// ragged: utterance b has mel_mask_lens[b] frames; mel and postnet_mel rows at or beyond it are zeroed.
static int decode_impl(const fs2_acoustic_model* m, const fs2_decode_args* a, cudaStream_t s, Arena& ar, bool ragged) {
  const int B = a->B, T = a->T, D = m->d_model;
  const size_t rows = (size_t)B * T;
  FftBufs f = fft_bufs(ar, m, rows, B, T, (m->tc_mask & FS2_TC_DECODER) != 0);
  int pc = 0;
  for (int i = 0; i < m->n_postnet; i++) pc = pc > m->post_cout[i] ? pc : m->post_cout[i];
  float* pa = ar.f32(rows * pc);
  float* pb = ar.f32(rows * pc);
  if (ar.dry) return FS2_OK;
  if (!f.x || !f.tmp || !f.qkv || !f.ctx || !f.hid || !pa || !pb || (f.att_bytes && !f.att_ws)) return FS2_ERR_WORKSPACE;
  if (T > m->dec_pos_rows) return FS2_ERR_ARG;

  const bool frame_level = m->pitch_frame_level || m->energy_frame_level;
  fs2_length_regulate_args lr{};
  lr.x = a->x_adapted; lr.cum = a->cum_dur; lr.pos = frame_level ? nullptr : m->dec_pos; lr.y = f.x; lr.B = B; lr.L = a->L; lr.T = T; lr.D = D;
  FS2_TRY(length_regulate(&lr, s));
  if (frame_level) {                                   // frame-level pitch / energy (model/modules.py:139-148), then the position add
    float* h1 = f.hid;                                 // [rows][d_inner] is free here and d_inner >= 2 * vp_filter is checked below
    float* h2 = f.hid + rows * m->vp_filter;
    if ((size_t)m->d_inner < 2 * (size_t)m->vp_filter) return FS2_ERR_UNSUPPORTED;
    fs2_variance_head_args v{};
    v.x = f.x; v.B = B; v.L = T; v.lens = a->mel_mask_lens; v.control = a->p_control;
    if (m->pitch_frame_level) {
      if (!a->p_pred_frames) return FS2_ERR_ARG;
      v.target = a->p_target_frames; v.bins = m->pitch_bins; v.emb = m->pitch_emb; v.pred_out = a->p_pred_frames;
      FS2_TRY(run_predictor(s, m, m->pitch, v, h1, h2, ragged));
    }
    if (m->energy_frame_level) {
      if (!a->e_pred_frames) return FS2_ERR_ARG;
      v.target = a->e_target_frames; v.bins = m->energy_bins; v.emb = m->energy_emb; v.pred_out = a->e_pred_frames;
      FS2_TRY(run_predictor(s, m, m->energy, v, h1, h2, ragged));
    }
    FS2_TRY(add_positions(f.x, m->dec_pos, B, T, D, s));
  }
  const ConvMode dec_mode{(m->tc_mask & FS2_TC_DECODER) ? ConvMode::TC : ConvMode::EXACT,
                          (m->tc_mask & FS2_TC_DECODER_F8) ? FS2_TC_VARIANT_F8 : 0u};
  for (int i = 0; i < m->n_dec; i++) FS2_TRY(fft_block(s, m, m->dec[i], f, B, T, a->mel_mask_lens, dec_mode, ragged));
  const ConvMode post_mode{(m->tc_mask & FS2_TC_POSTNET) ? ConvMode::TC : ConvMode::EXACT,
                           (m->tc_mask & FS2_TC_POSTNET_F8) ? FS2_TC_VARIANT_F8 : 0u};
  const int32_t* rag = ragged_lens(ragged, a->mel_mask_lens);
  fs2_conv1d_args c = conv_args(f.x, B, T, D, m->n_mel, 1, a->mel);
  post_mode.weights(c, m->w_mel, m->w_mel_tc, m->b_mel);
  c.x_lens = rag;
  FS2_TRY(conv1d_dispatch(&c, s));
  // PostNet: eval BatchNorm folded into (w, b) by the packer; unmasked, tanh on all but the last (Layers.py:129-137)
  const float* cur = a->mel;
  for (int i = 0; i < m->n_postnet; i++) {
    const bool last = i == m->n_postnet - 1;
    float* dst = last ? a->postnet_mel : ((i & 1) ? pb : pa);
    c = conv_args(cur, B, T, m->post_cin[i], m->post_cout[i], m->post_k, dst);
    post_mode.weights(c, m->w_post[i], m->w_post_tc[i], m->b_post[i]);
    if (last) c.res = a->mel;
    else c.out_act = FS2_ACT_TANH;
    c.x_lens = rag;
    FS2_TRY(conv1d_dispatch(&c, s));
    cur = dst;
  }
  if (ragged) return zero_tail(a->mel, a->postnet_mel, a->mel_mask_lens, B, T, m->n_mel, s);   // the convs left those rows unspecified
  return FS2_OK;
}

// ------------------------------------------------------------------ vocoder
// fs2_resstack arguments for stage i's ResBlock group on [B][N][C] rows: every kernel size and dilation, utterance b bounded by
// lens[b] * scale rows.  x, y, alpha and accumulate are the caller's (alpha 0: the kernel takes the mean over the n_kernels ResBlocks).
static fs2_resstack_args resblock_args(const fs2_vocoder_model* m, int i, int B, int N, int C, const int32_t* lens, int scale) {
  fs2_resstack_args a{};
  a.B = B; a.N = N; a.C = C; a.n_kernels = m->n_kernels; a.n_dil = m->n_dil;
  for (int j = 0; j < m->n_kernels; j++) {
    const int rb = i * m->n_kernels + j;
    a.k[j] = m->rb_k[j];
    for (int d = 0; d < m->n_dil; d++) {
      a.dil[j][d] = m->rb_dil[j][d];
      a.w1_tc[j][d] = m->w_rb1_tc[rb][d]; a.b1[j][d] = m->b_rb1[rb][d];
      a.w2_tc[j][d] = m->w_rb2_tc[rb][d]; a.b2[j][d] = m->b_rb2[rb][d];
    }
  }
  a.lens = lens; a.lens_scale = scale;
  return a;
}

// The same arguments narrowed to the one (dilated conv, conv) pair (j, d); fs2_resstack reads only the first n_kernels x n_dil entries.
static fs2_resstack_args resblock_pair(const fs2_resstack_args& g, int j, int d) {
  fs2_resstack_args a = g;
  a.n_kernels = 1; a.n_dil = 1;
  a.k[0] = g.k[j]; a.dil[0][0] = g.dil[j][d];
  a.w1_tc[0][0] = g.w1_tc[j][d]; a.b1[0][0] = g.b1[j][d];
  a.w2_tc[0][0] = g.w2_tc[j][d]; a.b2[0][0] = g.b2[j][d];
  return a;
}

static int vocoder_impl(const fs2_vocoder_model* m, const fs2_vocoder_args* a, cudaStream_t s, Arena& ar) {
  const int B = a->B, T = a->T;
  size_t per_frame = (size_t)m->c0;  // floats per mel frame of the widest activation
  {
    int up = 1, ch = m->c0;
    for (int i = 0; i < m->n_stages; i++) {
      up *= m->rates[i];
      ch /= 2;
      per_frame = per_frame > (size_t)up * ch ? per_frame : (size_t)up * ch;
    }
  }
  const size_t n = (size_t)B * T * per_frame;
  float* bx = ar.f32(n);
  float* bu = ar.f32(n);
  float* bt = ar.f32(n);
  float* r1 = ar.f32(n);
  float* r2 = ar.f32(n);
  if (ar.dry) return FS2_OK;
  if (!bx || !bu || !bt || !r1 || !r2) return FS2_ERR_WORKSPACE;
  // Ragged mode: every layer bounds utterance b by mel_lens[b] frames times its rows per mel frame (`scale`), so each utterance is
  // synthesised as if alone and the tiles of the padding are never computed.  Rows beyond an utterance are left unspecified in the
  // intermediates; conv_post writes them as zeros.
  const int32_t* lens = a->mel_lens;
  int scale = 1;

  // conv_pre reads the (possibly strided) channels-last mel view
  fs2_conv1d_args c = conv_args(a->mel, B, T, m->n_mel, m->c0, 7, bx);
  c.x_batch_stride = a->mel_batch_stride; c.x_row_stride = a->mel_row_stride;
  c.res_batch_stride = c.res_row_stride = 0;                        // no residual
  c.w = m->w_pre; c.w_tc = m->w_pre_tc; c.bias = m->b_pre; c.tc_variant = (m->f8_mask & 1) ? FS2_TC_VARIANT_F8 : 0;
  c.x_lens = lens; c.lens_scale = scale;
  FS2_TRY(conv1d_dispatch(&c, s));
  int Ti = T, C = m->c0;
  const float inv_nk = 1.f / (float)m->n_kernels;
  for (int i = 0; i < m->n_stages; i++) {
    const int u = m->rates[i], Co = C / 2;
    if (m->up_k[i] != 2 * u || (u & 1)) return FS2_ERR_UNSUPPORTED;
    const unsigned tcv = (m->f8_mask & (2 << i)) ? FS2_TC_VARIANT_F8 : 0;
    // ---- lrelu + ConvTranspose1d as two 2-tap phase-group convolutions (hifigan/models.py:152-153)
    for (int g = 0; g < 2; g++) {
      const size_t off = (size_t)g * (u / 2) * Co;    // group g writes output channels [off, off + (u/2)*Co) of each [u*Co] row
      c = conv_args(bx, B, Ti, C, (u / 2) * Co, 2, bu + off);
      c.y_batch_stride = (int64_t)Ti * u * Co; c.y_row_stride = (int64_t)u * Co;
      c.res_batch_stride = c.res_row_stride = 0;                    // no residual
      c.pad_left = g == 0 ? 1 : 0;
      c.w = g == 0 ? m->w_up_a[i] : m->w_up_b[i];
      c.w_tc = g == 0 ? m->w_up_a_tc[i] : m->w_up_b_tc[i];
      c.bias = m->b_up[i] + off;
      c.in_act = FS2_ACT_LRELU; c.in_slope = 0.1f; c.tc_variant = tcv;
      c.x_lens = lens; c.lens_scale = scale;          // [B][Ti][u*Co]: input and output rows have the same n_b
      FS2_TRY(conv1d_dispatch(&c, s));
    }
    Ti *= u; C = Co; scale *= u;
    // ---- mean of the multi-receptive-field ResBlocks (models.py:154-160, ResBlock.forward :96-103)
    fs2_resstack_args group = resblock_args(m, i, B, Ti, C, lens, scale);
    if ((m->fused_mask >> i) & 1) {                    // one persistent kernel for the whole group: intermediates never leave the SM
      if (!tcv) return FS2_ERR_ARG;
      group.x = bu; group.y = bx;
      FS2_TRY(resstack(&group, s));
      continue;
    }
    for (int j = 0; j < m->n_kernels; j++) {
      const int rb = i * m->n_kernels + j, k = m->rb_k[j];
      const float* r = bu;
      const bool pairs = ((m->pair_mask >> i) & 1) && tcv && (C == 32 || C == 64) && k <= m->pair_kmax;
      for (int d = 0; d < m->n_dil; d++) {
        const bool last = d == m->n_dil - 1;            // the last layer adds its share of the mean over the n_kernels ResBlocks into bx
        float* dst = last ? bx : (r == r1 ? r2 : r1);
        const float alpha = last ? inv_nk : 1.f;
        const int accumulate = last && j > 0;
        if (pairs) {                                   // one launch per (dilated conv, conv, +x) pair: the intermediate stays on chip
          fs2_resstack_args p = resblock_pair(group, j, d);
          p.x = r; p.y = dst; p.alpha = alpha; p.accumulate = accumulate;
          FS2_TRY(resstack(&p, s));
        } else {                                       // the two convs through bt
          const int dil = m->rb_dil[j][d];
          c = conv_args(r, B, Ti, C, C, k, bt);
          c.w = m->w_rb1[rb][d]; c.w_tc = m->w_rb1_tc[rb][d]; c.bias = m->b_rb1[rb][d]; c.tc_variant = tcv;
          c.dilation = dil; c.pad_left = (k * dil - dil) / 2;
          c.in_act = c.out_act = FS2_ACT_LRELU; c.in_slope = c.out_slope = 0.1f;
          c.x_lens = lens; c.lens_scale = scale;
          FS2_TRY(conv1d_dispatch(&c, s));
          c = conv_args(bt, B, Ti, C, C, k, dst);
          c.w = m->w_rb2[rb][d]; c.w_tc = m->w_rb2_tc[rb][d]; c.bias = m->b_rb2[rb][d]; c.tc_variant = tcv;
          c.res = r; c.alpha = alpha; c.accumulate = accumulate;
          c.x_lens = lens; c.lens_scale = scale;
          FS2_TRY(conv1d_dispatch(&c, s));
        }
        r = dst;
      }
    }
  }
  fs2_conv_post_args p{};
  p.x = bx; p.B = B; p.T = Ti; p.C = C; p.w = m->w_post; p.bias = m->b_post; p.taps = 7; p.in_slope = 0.01f; p.wav = a->wav;
  p.lens = lens; p.lens_scale = scale;
  return conv_post(&p, s);
}

}  // namespace fs2

// ====================================================================== extern "C"
using namespace fs2;
#define S(x) ((cudaStream_t)(x))

extern "C" {

int fs2_abi_version(void) { return 11; }
int fs2_conv_tc_block(int N) { return conv_tc_nb(N, 128); }
int fs2_conv_tc_block_f8(int N) { return conv_tc_nb(N, 64); }
int fs2_conv_tc_plan(const fs2_conv1d_args* a, int num_sms, int32_t* out) { return conv_tc_plan_query(a, num_sms, out); }
int64_t fs2_kernel_launch_count(void) { return (int64_t)g_launch_count.load(); }
size_t fs2_struct_size(int which) {
  switch (which) {
    case 0: return sizeof(fs2_conv1d_args);
    case 1: return sizeof(fs2_layernorm_args);
    case 2: return sizeof(fs2_attention_args);
    case 3: return sizeof(fs2_embed_args);
    case 4: return sizeof(fs2_rowbias_args);
    case 5: return sizeof(fs2_variance_head_args);
    case 6: return sizeof(fs2_durations_args);
    case 7: return sizeof(fs2_length_regulate_args);
    case 8: return sizeof(fs2_conv_post_args);
    case 9: return sizeof(fs2_acoustic_model);
    case 10: return sizeof(fs2_encode_args);
    case 11: return sizeof(fs2_decode_args);
    case 12: return sizeof(fs2_vocoder_model);
    case 13: return sizeof(fs2_vocoder_args);
    case 14: return sizeof(fs2_resstack_args);
    case 15: return sizeof(fs2_wav_int16_args);
    default: return 0;
  }
}
int fs2_profile_begin(void) {
  g_prof.clear();
  g_prof_on = true;
  return FS2_OK;
}
int fs2_profile_end(double* ms, double* flops, int64_t* launches) {
  g_prof_on = false;
  if (!ms || !flops || !launches) return FS2_ERR_ARG;
  for (int i = 0; i < FS2_PROF_CLASSES; i++) { ms[i] = 0; flops[i] = 0; launches[i] = 0; }
  int rc = FS2_OK;
  for (auto& r : g_prof) {
    float t = 0.f;
    cudaError_t e = cudaEventSynchronize(r.b);
    if (e == cudaSuccess) e = cudaEventElapsedTime(&t, r.a, r.b);
    if (e != cudaSuccess) rc = FS2_ERR_CUDA - (int)e;
    const int c = (r.cls >= 0 && r.cls < FS2_PROF_CLASSES) ? r.cls : 3;
    ms[c] += t; flops[c] += r.flops; launches[c] += 1;
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  g_prof.clear();
  return rc;
}
const char* fs2_build_info(void) { return "fs2b200 sm_90a (wgmma split-FP16 conv + attention, fp32 CUDA-core kernels), built " __DATE__ " " __TIME__; }

int fs2_conv1d(const fs2_conv1d_args* a, fs2_stream_t st) { return conv1d_dispatch(a, S(st)); }
int fs2_layernorm(const fs2_layernorm_args* a, fs2_stream_t st) { return layernorm(a, S(st)); }
int fs2_attention(const fs2_attention_args* a, fs2_stream_t st) {
  if (!a) return FS2_ERR_ARG;
  if (a->backend == 0) return attention_simt(a, S(st));
  if (a->backend == 2) return attention_fused(a, a->workspace, a->workspace_bytes, S(st));
  return FS2_ERR_ARG;
}
size_t fs2_attention_workspace_bytes(int B, int T, int H) {      // backend 2
  if (!(B > 0 && T > 0 && H > 0)) return 0;
  return attention_fused_workspace(B, T, H);
}
int fs2_embed_positions(const fs2_embed_args* a, fs2_stream_t st) { return embed_positions(a, S(st)); }
int fs2_add_speaker(const fs2_rowbias_args* a, fs2_stream_t st) { return add_speaker(a, S(st)); }
int fs2_variance_head(const fs2_variance_head_args* a, fs2_stream_t st) { return variance_head(a, S(st)); }
int fs2_durations(const fs2_durations_args* a, fs2_stream_t st) { return durations(a, S(st)); }
int fs2_length_regulate(const fs2_length_regulate_args* a, fs2_stream_t st) { return length_regulate(a, S(st)); }
int fs2_conv_post(const fs2_conv_post_args* a, fs2_stream_t st) { return conv_post(a, S(st)); }
int fs2_resstack(const fs2_resstack_args* a, fs2_stream_t st) { return resstack(a, S(st)); }
int fs2_wav_to_int16(const fs2_wav_int16_args* a, fs2_stream_t st) { return wav_to_int16(a, S(st)); }
int fs2_resstack_plan(const fs2_resstack_args* a, int num_sms, int32_t* out) { return out ? resstack_plan(a, num_sms, out) : FS2_ERR_ARG; }
int fs2_add_positions(float* x, const float* pos, int B, int T, int D, fs2_stream_t st) { return add_positions(x, pos, B, T, D, S(st)); }
int fs2_transpose_bct_to_btc(const float* in, float* out, int B, int C, int T, fs2_stream_t st) {
  return transpose_bct_to_btc(in, out, B, C, T, S(st));
}

size_t fs2_encode_workspace_bytes(const fs2_acoustic_model* m, int B, int L) {
  if (!model_ok(m) || B <= 0 || L <= 0) return 0;
  Arena ar(nullptr, 0);
  fs2_encode_args a{};
  a.B = B; a.L = L;
  encode_impl(m, &a, nullptr, ar, false);
  return ar.off + 256;
}

static int acoustic_encode(const fs2_acoustic_model* m, const fs2_encode_args* a, fs2_stream_t st, bool ragged) {
  if (!model_ok(m) || !a || a->B <= 0 || a->L <= 0) return FS2_ERR_ARG;
  if (!a->texts || !a->src_lens || !a->logd_pred || !a->mel_lens || !a->cum_dur || !a->x_adapted ||
      !a->len_stats || !a->workspace)
    return FS2_ERR_ARG;
  if (!a->d_target && !a->d_rounded) return FS2_ERR_ARG;
  if (m->d_model / m->n_head != 128) return FS2_ERR_UNSUPPORTED;
  Arena ar(a->workspace, a->workspace_bytes);
  return encode_impl(m, a, S(st), ar, ragged);
}
int fs2_acoustic_encode(const fs2_acoustic_model* m, const fs2_encode_args* a, fs2_stream_t st) { return acoustic_encode(m, a, st, false); }
int fs2_acoustic_encode_ragged(const fs2_acoustic_model* m, const fs2_encode_args* a, fs2_stream_t st) { return acoustic_encode(m, a, st, true); }

size_t fs2_decode_workspace_bytes(const fs2_acoustic_model* m, int B, int T) {
  if (!model_ok(m) || B <= 0 || T <= 0) return 0;
  Arena ar(nullptr, 0);
  fs2_decode_args a{};
  a.B = B; a.T = T;
  decode_impl(m, &a, nullptr, ar, false);
  return ar.off + 256;
}

static int acoustic_decode(const fs2_acoustic_model* m, const fs2_decode_args* a, fs2_stream_t st, bool ragged) {
  if (!model_ok(m) || !a || a->B <= 0 || a->L <= 0 || a->T <= 0) return FS2_ERR_ARG;
  if (!a->x_adapted || !a->cum_dur || !a->mel_mask_lens || !a->mel || !a->postnet_mel || !a->workspace) return FS2_ERR_ARG;
  if (m->d_model / m->n_head != 128) return FS2_ERR_UNSUPPORTED;
  Arena ar(a->workspace, a->workspace_bytes);
  return decode_impl(m, a, S(st), ar, ragged);
}
int fs2_acoustic_decode(const fs2_acoustic_model* m, const fs2_decode_args* a, fs2_stream_t st) { return acoustic_decode(m, a, st, false); }
int fs2_acoustic_decode_ragged(const fs2_acoustic_model* m, const fs2_decode_args* a, fs2_stream_t st) { return acoustic_decode(m, a, st, true); }

static bool vocoder_ok(const fs2_vocoder_model* m) {
  if (!(m && m->n_stages > 0 && m->n_stages <= FS2_MAX_STAGES && m->n_kernels > 0 && m->n_kernels <= FS2_MAX_DIL + 4 &&
        m->n_kernels * m->n_stages <= FS2_MAX_RESBLOCKS && m->n_dil > 0 && m->n_dil <= FS2_MAX_DIL && m->c0 > 0 && m->n_mel > 0))
    return false;
  if (m->c0 % (1 << m->n_stages)) return false;                          // channels halve at every stage
  for (int i = 0; i < m->n_stages; i++)
    if (m->rates[i] <= 0 || m->up_k[i] <= 0) return false;
  for (int j = 0; j < m->n_kernels; j++) {
    if (m->rb_k[j] <= 0 || !(m->rb_k[j] & 1)) return false;              // odd kernels: symmetric "same" padding (hifigan/models.py:16-17)
    for (int d = 0; d < m->n_dil; d++)
      if (m->rb_dil[j][d] <= 0) return false;
  }
  return true;
}

size_t fs2_vocoder_workspace_bytes(const fs2_vocoder_model* m, int B, int T) {
  if (!vocoder_ok(m) || B <= 0 || T <= 0) return 0;
  Arena ar(nullptr, 0);
  fs2_vocoder_args a{};
  a.B = B; a.T = T;
  vocoder_impl(m, &a, nullptr, ar);
  return ar.off + 256;
}

int fs2_vocoder_forward(const fs2_vocoder_model* m, const fs2_vocoder_args* a, fs2_stream_t st) {
  if (!vocoder_ok(m) || !a || a->B <= 0 || a->T <= 0 || !a->mel || !a->wav || !a->workspace) return FS2_ERR_ARG;
  Arena ar(a->workspace, a->workspace_bytes);
  return vocoder_impl(m, a, S(st), ar);
}

}  // extern "C"
