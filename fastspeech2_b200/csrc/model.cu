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
// win: the vocoder's windowed mode (OriginWindow), NULL everywhere else.  lw / vr: the table mode (LaunchWeights, VoiceRow: the
// multi-generator pool, the acoustic voices mode), NULL everywhere else
int conv1d_simt(const fs2_conv1d_args* a, cudaStream_t s, const OriginWindow* win = nullptr, const LaunchWeights* lw = nullptr);
int conv_simt_plan(const fs2_conv1d_args* a, int num_sms, fs2_conv_simt_plan_t* out);
int conv1d_tc(const fs2_conv1d_args* a, cudaStream_t s, const OriginWindow* win = nullptr, const LaunchWeights* lw = nullptr);
int attention_fused(const fs2_attention_args* a, void* ws, size_t ws_bytes, cudaStream_t s, bool ragged = false);
size_t attention_fused_workspace(int B, int T, int H);
bool conv_tc_supported(const fs2_conv1d_args* a);
int conv_tc_nb(int N, int nb_max);
int conv_tc_plan_query(const fs2_conv1d_args* a, int num_sms, fs2_conv_tc_plan_t* out);

// backend dispatch of the fs2_conv1d contract
static int conv1d_dispatch(const fs2_conv1d_args* a, cudaStream_t s, const OriginWindow* win = nullptr, const LaunchWeights* lw = nullptr) {
  if (!a) return FS2_ERR_ARG;
  if (a->x_lens && a->lens_scale < 1) return FS2_ERR_ARG;
  if (a->backend == FS2_CONV_TC) return conv1d_tc(a, s, win, lw);
  if (a->backend == FS2_CONV_AUTO && a->w_tc && conv_tc_supported(a)) return conv1d_tc(a, s, win, lw);
  return conv1d_simt(a, s, win, lw);
}
int attention_simt(const fs2_attention_args* a, cudaStream_t s, bool ragged = false, int fused_from = 0);
int embed_positions(const fs2_embed_args* a, cudaStream_t s, const VoiceRow* vr = nullptr);
int add_speaker(const fs2_rowbias_args* a, cudaStream_t s, const VoiceRow* vr = nullptr);
int layernorm(const fs2_layernorm_args* a, cudaStream_t s, const VoiceRow* vr = nullptr);
int variance_head(const fs2_variance_head_args* a, cudaStream_t s, const ControlView* ctl = nullptr, const VoiceRow* vr = nullptr);
int durations(const fs2_durations_args* a, cudaStream_t s, const int32_t* src_lens = nullptr, const ControlView* ctl = nullptr,
              const int32_t* valid = nullptr);
int length_regulate(const fs2_length_regulate_args* a, cudaStream_t s, const VoiceRow* vr = nullptr);
int conv_post(const fs2_conv_post_args* a, cudaStream_t s, const OriginWindow* win = nullptr, const LaunchWeights* lw = nullptr,
              long long x_bs = 0, long long wav_bs = 0);
int resstack(const fs2_resstack_args* a, cudaStream_t s, const OriginWindow* win = nullptr, const LaunchWeights* lw = nullptr, int x0 = 0,
             bool wide = false);
int stage_mel(const MelSource& src, int B, int x0, int rows, int n_mel, float* out, int32_t* org, int32_t* lens, const int32_t* gen_in,
              int n_gen, int32_t* gen, cudaStream_t s);
int mel_ring_append(const fs2_mel_ring_append_args* a, cudaStream_t s);
int wav_to_int16(const fs2_wav_int16_args* a, cudaStream_t s);
int resstack_plan(const fs2_resstack_args* a, int num_sms, fs2_resstack_plan_t& out, bool wide = false);
int transpose_bct_to_btc(const float* in, float* out, int B, int C, int T, cudaStream_t s);
int add_positions(float* x, const float* pos, int B, int T, int D, cudaStream_t s, const VoiceRow* vr = nullptr);
int zero_tail(float* y0, float* y1, const int32_t* lens, int B, int T, int C, cudaStream_t s);

// The table mode (ModelTable): the device array of models M and the staged table of each row's model, and a field's ref relative to
// model 0 (m)
template <class M>
static ModelTable model_table(const M* models_dev, const int32_t* sel) {
  return ModelTable{reinterpret_cast<const unsigned char*>(models_dev), sel, (int)sizeof(M)};
}
template <class M>
static FieldRef field_ref(const M* m, const void* field, int add = 0) {
  return FieldRef{(int32_t)((const char*)field - (const char*)m), add};
}

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
// The voices mode (fs2_acoustic_{encode,decode}_voices): the phase plans and checks on m = models[0] and names each weight a launch reads
// by its field in *m; utterance b reads that field of voice staged[b] of models_dev.  staged: the phase's [2B] table (VoiceRow::out),
// staged from the caller's `in` by the phase's first launch.  Each launch's VoiceRow / LaunchWeights is built right before it.
struct VoiceSet {
  const fs2_acoustic_model* m;
  const fs2_acoustic_model* models_dev;
  int32_t* staged;
  const int32_t* in; int n;
  mutable VoiceRow vr;
  mutable LaunchWeights lw;
  FieldRef ref(const void* field) const { return field ? field_ref(m, field) : FieldRef{}; }
  const VoiceRow* row(const void* f0, const void* f1 = nullptr, const void* f2 = nullptr, const void* f3 = nullptr, bool first = false) const {
    vr = VoiceRow{model_table(models_dev, staged), {ref(f0), ref(f1), ref(f2), ref(f3)}, first ? in : nullptr, n, first ? staged : nullptr};
    return &vr;
  }
  const LaunchWeights* conv(const void* w, const void* w_tc, const void* bias) const {
    lw = LaunchWeights{model_table(models_dev, staged), ref(w), ref(w_tc), ref(bias), 0, 0};
    return &lw;
  }
};
// The row tables of a launch: NULL outside the voices mode
template <class... F>
static const VoiceRow* voice_row(const VoiceSet* vs, F... fields) { return vs ? vs->row(fields...) : nullptr; }

struct ConvMode {
  enum { EXACT, TC, SEGMENTED } path;
  unsigned tcv;
  const VoiceSet* vs;     // the voices mode, or NULL
  // Runs `a` with these weights (fields of the model: in the voices mode each utterance reads them from its own voice).
  int run(fs2_conv1d_args& a, const float* const& w, const float* const& w_tc, const float* const& bias, cudaStream_t s) const {
    a.bias = bias;
    if (path == SEGMENTED) {
      a.w = nullptr; a.w_tc = w_tc; a.backend = FS2_CONV_TC; a.tc_variant = FS2_TC_VARIANT_NB64 | FS2_TC_VARIANT_SEGMENTED;
    } else {
      a.w = w; a.w_tc = path == TC ? w_tc : nullptr; a.tc_variant = tcv;
    }
    return conv1d_dispatch(&a, s, nullptr, vs ? vs->conv(&w, &w_tc, &bias) : nullptr);
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
  c.x_lens = rag;
  FS2_TRY(mode.run(c, w.w_qkv, w.w_qkv_tc, w.b_qkv, s));
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
  c.res = f.x;
  c.x_lens = rag;
  FS2_TRY(mode.run(c, w.w_o, w.w_o_tc, w.b_o, s));
  fs2_layernorm_args n{};                                           // both LayerNorms: tmp -> x, padded rows zeroed
  n.x = f.tmp; n.y = f.x; n.B = B; n.T = T; n.C = D; n.eps = 1e-5f; n.row_lens = lens;
  n.gamma = w.ln1_g; n.beta = w.ln1_b;
  FS2_TRY(layernorm(&n, s, voice_row(mode.vs, &w.ln1_g, &w.ln1_b)));
  // conv-FFN.  K-segmented: w_1 leaves the pre-activation hidden and the ReLU is w_2's input activation (leaky_relu with slope 0)
  c = conv_args(f.x, B, T, D, F, m->k1, f.hid);
  if (!seg) c.out_act = FS2_ACT_RELU;
  c.x_lens = rag;
  FS2_TRY(mode.run(c, w.w_1, w.w_1_tc, w.b_1, s));
  c = conv_args(f.hid, B, T, F, D, m->k2, f.tmp);
  c.res = f.x;
  if (seg) { c.in_act = FS2_ACT_LRELU; c.in_slope = 0.f; }
  c.x_lens = rag;
  FS2_TRY(mode.run(c, w.w_2, w.w_2_tc, w.b_2, s));
  n.gamma = w.ln2_g; n.beta = w.ln2_b;
  return layernorm(&n, s, voice_row(mode.vs, &w.ln2_g, &w.ln2_b));
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
// ctl: the per-element control that replaces head.control (ctl.v NULL: the scalar).  vs: the voices mode, or NULL (w is then one of m's
// predictors, and head.bins / head.emb m's tables of the same quantity).
static int run_predictor(cudaStream_t s, const fs2_acoustic_model* m, const fs2_predictor_weights& w, fs2_variance_head_args head,
                         float* h1, float* h2, bool ragged, const ControlView& ctl, const VoiceSet* vs) {
  const int B = head.B, T = head.L, k = m->vp_kernel, D = m->d_model, VF = m->vp_filter;
  const bool seg = (m->tc_mask & FS2_TC_PREDICTORS) && w.w_c1_tc && w.w_c2_tc;   // K-segmented: the ReLU is applied by the LayerNorm
  const ConvMode mode{seg ? ConvMode::SEGMENTED : ConvMode::EXACT, 0, vs};
  const int32_t* rag = ragged_lens(ragged, head.lens);
  fs2_layernorm_args n{};                                           // both LayerNorms: h1 -> h2, unmasked (ragged: masked)
  n.x = h1; n.y = h2; n.B = B; n.T = T; n.C = VF; n.eps = 1e-5f; n.pre_relu = seg; n.row_lens = rag;
  fs2_conv1d_args c = conv_args(head.x, B, T, D, VF, k, h1);
  if (!seg) c.out_act = FS2_ACT_RELU;
  c.x_lens = rag;
  FS2_TRY(mode.run(c, w.w_c1, w.w_c1_tc, w.b_c1, s));
  n.gamma = w.ln1_g; n.beta = w.ln1_b;
  FS2_TRY(layernorm(&n, s, voice_row(vs, &w.ln1_g, &w.ln1_b)));
  c = conv_args(h2, B, T, VF, VF, k, h1);
  c.pad_left = 1;                                                   // padding=1 is hard-coded upstream
  if (!seg) c.out_act = FS2_ACT_RELU;
  c.x_lens = rag;
  FS2_TRY(mode.run(c, w.w_c2, w.w_c2_tc, w.b_c2, s));
  n.gamma = w.ln2_g; n.beta = w.ln2_b;
  FS2_TRY(layernorm(&n, s, voice_row(vs, &w.ln2_g, &w.ln2_b)));
  head.h = h2; head.w = w.w_out; head.b = w.b_out; head.C = VF; head.n_edges = m->n_bins - 1; head.D = D;
  const bool pitch = &w == &m->pitch;                              // the bins and embedding of the predictor's quantity (none: durations)
  return variance_head(&head, s, &ctl, voice_row(vs, &w.w_out, &w.b_out, pitch ? &m->pitch_bins : &m->energy_bins,
                                                 pitch ? &m->pitch_emb : &m->energy_emb));
}

// The p (pitch / energy) or d (durations) control of fs2_control_args on the phase's [B][L] rows; ragged: columns l >= lens[b] are not read.
static ControlView control_view(const float* v, int64_t sb, int64_t sl, bool ragged, const int32_t* lens) {
  return ControlView{v, sb, sl, v ? ragged_lens(ragged, lens) : nullptr};
}

// ------------------------------------------------------------------ phase 1
// ragged: utterance b has src_lens[b] phonemes; x_adapted rows at or beyond it are left unspecified.
// ctl: NULL, or the per-element p / d controls that replace a->p_control / a->d_control where their pointers are set.
// voices: NULL, or the voices mode (m = voices->models[0]): the staged table is the workspace's first allocation, so the workspace is the
// single model's plus that table.
static int encode_impl(const fs2_acoustic_model* m, const fs2_encode_args* a, const fs2_control_args* ctl, cudaStream_t s, Arena& ar,
                       bool ragged, const fs2_acoustic_voices* voices = nullptr) {
  const int B = a->B, L = a->L, D = m->d_model, VF = m->vp_filter;
  const size_t rows = (size_t)B * L;
  int32_t* staged = voices ? (int32_t*)ar.take((size_t)2 * B * sizeof(int32_t)) : nullptr;
  FftBufs f = fft_bufs(ar, m, rows);
  float* h1 = ar.f32(rows * VF);
  float* h2 = ar.f32(rows * VF);
  if (ar.dry) return FS2_OK;
  if (!f.x || !f.tmp || !f.qkv || !f.ctx || !f.hid || !h1 || !h2 || (voices && !staged)) return FS2_ERR_WORKSPACE;
  if (L > m->enc_pos_rows) return FS2_ERR_ARG;
  const VoiceSet vset{m, voices ? voices->models_dev : nullptr, staged, voices ? voices->voice : nullptr, voices ? voices->n : 0, {}, {}};
  const VoiceSet* vs = voices ? &vset : nullptr;

  fs2_embed_args e{};
  e.ids = a->texts; e.table = m->word_emb; e.pos = m->enc_pos; e.y = f.x; e.B = B; e.L = L; e.D = D; e.n_vocab = m->n_vocab;
  FS2_TRY(embed_positions(&e, s, vs ? vs->row(&m->word_emb, &m->enc_pos, nullptr, nullptr, true) : nullptr));
  const ConvMode enc_mode{(m->tc_mask & FS2_TC_ENCODER) ? ConvMode::SEGMENTED : ConvMode::EXACT, 0, vs};   // exact attention either way
  for (int i = 0; i < m->n_enc; i++) FS2_TRY(fft_block(s, m, m->enc[i], f, B, L, a->src_lens, enc_mode, ragged));
  if (m->spk_emb) {
    if (!a->speakers) return FS2_ERR_ARG;
    fs2_rowbias_args r{};
    r.x = f.x; r.table = m->spk_emb; r.idx = a->speakers; r.B = B; r.L = L; r.D = D; r.n_rows = m->n_speakers;
    FS2_TRY(add_speaker(&r, s, voice_row(vs, &m->spk_emb)));
  }
  // x_adapted starts as the encoder output; pitch / energy embeddings are added in place (modules.py:117-126)
  cudaError_t ce = cudaMemcpyAsync(a->x_adapted, f.x, rows * D * sizeof(float), cudaMemcpyDeviceToDevice, s);
  if (ce != cudaSuccess) return FS2_ERR_CUDA - (int)ce;

  // duration on the un-embedded x; pitch on x; energy on x + pitch embedding.  energy uses p_control (modules.py:124).
  fs2_variance_head_args v{};
  v.x = a->x_adapted; v.B = B; v.L = L; v.lens = a->src_lens; v.control = 1.f; v.pred_out = a->logd_pred;
  FS2_TRY(run_predictor(s, m, m->dur, v, h1, h2, ragged, ControlView{}, vs));
  v.control = a->p_control;
  const ControlView p_ctl = ctl ? control_view(ctl->p, ctl->p_stride_b, ctl->p_stride_l, ragged, a->src_lens) : ControlView{};
  if (!m->pitch_frame_level) {
    if (!a->p_pred) return FS2_ERR_ARG;
    v.target = a->p_target; v.bins = m->pitch_bins; v.emb = m->pitch_emb; v.pred_out = a->p_pred;
    FS2_TRY(run_predictor(s, m, m->pitch, v, h1, h2, ragged, p_ctl, vs));
  }
  if (!m->energy_frame_level) {
    if (!a->e_pred) return FS2_ERR_ARG;
    v.target = a->e_target; v.bins = m->energy_bins; v.emb = m->energy_emb; v.pred_out = a->e_pred;
    FS2_TRY(run_predictor(s, m, m->energy, v, h1, h2, ragged, p_ctl, vs));
  }

  fs2_durations_args d{};
  d.src = a->d_target ? a->d_target : a->logd_pred; d.use_target = a->d_target != nullptr; d.d_control = a->d_control;
  d.B = B; d.L = L; d.d_rounded = a->d_target ? nullptr : a->d_rounded; d.cum = a->cum_dur; d.mel_lens = a->mel_lens;
  d.mel_lens32 = a->mel_lens32; d.len_stats = a->len_stats;
  const ControlView d_ctl = ctl ? control_view(ctl->d, ctl->d_stride_b, ctl->d_stride_l, ragged, a->src_lens) : ControlView{};
  FS2_TRY(durations(&d, s, ragged_lens(ragged, a->src_lens), &d_ctl, vs ? staged + B : nullptr));
  if (a->len_stats_host) {
    ce = cudaMemcpyAsync(a->len_stats_host, a->len_stats, 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
    if (ce != cudaSuccess) return FS2_ERR_CUDA - (int)ce;
  }
  return FS2_OK;
}

// ------------------------------------------------------------------ phase 2
// ragged: utterance b has mel_mask_lens[b] frames; mel and postnet_mel rows at or beyond it are zeroed.
// ctl: NULL, or the per-frame p control that replaces a->p_control when ctl->p is set (ctl->d is not read).
// voices: NULL, or the voices mode, as in encode_impl.
static int decode_impl(const fs2_acoustic_model* m, const fs2_decode_args* a, const fs2_control_args* ctl, cudaStream_t s, Arena& ar,
                       bool ragged, const fs2_acoustic_voices* voices = nullptr) {
  const int B = a->B, T = a->T, D = m->d_model;
  const size_t rows = (size_t)B * T;
  int32_t* staged = voices ? (int32_t*)ar.take((size_t)2 * B * sizeof(int32_t)) : nullptr;
  FftBufs f = fft_bufs(ar, m, rows, B, T, (m->tc_mask & FS2_TC_DECODER) != 0);
  int pc = 0;
  for (int i = 0; i < m->n_postnet; i++) pc = pc > m->post_cout[i] ? pc : m->post_cout[i];
  float* pa = ar.f32(rows * pc);
  float* pb = ar.f32(rows * pc);
  if (ar.dry) return FS2_OK;
  if (!f.x || !f.tmp || !f.qkv || !f.ctx || !f.hid || !pa || !pb || (f.att_bytes && !f.att_ws) || (voices && !staged)) return FS2_ERR_WORKSPACE;
  if (T > m->dec_pos_rows) return FS2_ERR_ARG;
  const VoiceSet vset{m, voices ? voices->models_dev : nullptr, staged, voices ? voices->voice : nullptr, voices ? voices->n : 0, {}, {}};
  const VoiceSet* vs = voices ? &vset : nullptr;

  const bool frame_level = m->pitch_frame_level || m->energy_frame_level;
  fs2_length_regulate_args lr{};
  lr.x = a->x_adapted; lr.cum = a->cum_dur; lr.pos = frame_level ? nullptr : m->dec_pos; lr.y = f.x; lr.B = B; lr.L = a->L; lr.T = T; lr.D = D;
  FS2_TRY(length_regulate(&lr, s, vs ? vs->row(&m->dec_pos, nullptr, nullptr, nullptr, true) : nullptr));
  if (frame_level) {                                   // frame-level pitch / energy (model/modules.py:139-148), then the position add
    float* h1 = f.hid;                                 // [rows][d_inner] is free here and d_inner >= 2 * vp_filter is checked below
    float* h2 = f.hid + rows * m->vp_filter;
    if ((size_t)m->d_inner < 2 * (size_t)m->vp_filter) return FS2_ERR_UNSUPPORTED;
    fs2_variance_head_args v{};
    v.x = f.x; v.B = B; v.L = T; v.lens = a->mel_mask_lens; v.control = a->p_control;
    const ControlView p_ctl = ctl ? control_view(ctl->p, ctl->p_stride_b, ctl->p_stride_l, ragged, a->mel_mask_lens) : ControlView{};
    if (m->pitch_frame_level) {
      if (!a->p_pred_frames) return FS2_ERR_ARG;
      v.target = a->p_target_frames; v.bins = m->pitch_bins; v.emb = m->pitch_emb; v.pred_out = a->p_pred_frames;
      FS2_TRY(run_predictor(s, m, m->pitch, v, h1, h2, ragged, p_ctl, vs));
    }
    if (m->energy_frame_level) {
      if (!a->e_pred_frames) return FS2_ERR_ARG;
      v.target = a->e_target_frames; v.bins = m->energy_bins; v.emb = m->energy_emb; v.pred_out = a->e_pred_frames;
      FS2_TRY(run_predictor(s, m, m->energy, v, h1, h2, ragged, p_ctl, vs));
    }
    FS2_TRY(add_positions(f.x, m->dec_pos, B, T, D, s, voice_row(vs, &m->dec_pos)));
  }
  const ConvMode dec_mode{(m->tc_mask & FS2_TC_DECODER) ? ConvMode::TC : ConvMode::EXACT,
                          (m->tc_mask & FS2_TC_DECODER_F8) ? FS2_TC_VARIANT_F8 : 0u, vs};
  for (int i = 0; i < m->n_dec; i++) FS2_TRY(fft_block(s, m, m->dec[i], f, B, T, a->mel_mask_lens, dec_mode, ragged));
  const ConvMode post_mode{(m->tc_mask & FS2_TC_POSTNET) ? ConvMode::TC : ConvMode::EXACT,
                           (m->tc_mask & FS2_TC_POSTNET_F8) ? FS2_TC_VARIANT_F8 : 0u, vs};
  const int32_t* rag = ragged_lens(ragged, a->mel_mask_lens);
  fs2_conv1d_args c = conv_args(f.x, B, T, D, m->n_mel, 1, a->mel);
  c.x_lens = rag;
  FS2_TRY(post_mode.run(c, m->w_mel, m->w_mel_tc, m->b_mel, s));
  // PostNet: eval BatchNorm folded into (w, b) by the packer; unmasked, tanh on all but the last (Layers.py:129-137)
  const float* cur = a->mel;
  for (int i = 0; i < m->n_postnet; i++) {
    const bool last = i == m->n_postnet - 1;
    float* dst = last ? a->postnet_mel : ((i & 1) ? pb : pa);
    c = conv_args(cur, B, T, m->post_cin[i], m->post_cout[i], m->post_k, dst);
    if (last) c.res = a->mel;
    else c.out_act = FS2_ACT_TANH;
    c.x_lens = rag;
    FS2_TRY(post_mode.run(c, m->w_post[i], m->w_post_tc[i], m->b_post[i], s));
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

// The same arguments narrowed to ResBlock j's (dilated conv, conv) pairs [d0, d1); fs2_resstack reads only the first n_kernels x n_dil
// entries.
static fs2_resstack_args resblock_run(const fs2_resstack_args& g, int j, int d0, int d1) {
  fs2_resstack_args a = g;
  a.n_kernels = 1; a.n_dil = d1 - d0;
  a.k[0] = g.k[j];
  for (int d = d0; d < d1; d++) {
    a.dil[0][d - d0] = g.dil[j][d];
    a.w1_tc[0][d - d0] = g.w1_tc[j][d]; a.b1[0][d - d0] = g.b1[j][d];
    a.w2_tc[0][d - d0] = g.w2_tc[j][d]; a.b2[0][d - d0] = g.b2[j][d];
  }
  return a;
}

static bool resstack_width(int C) { return C == 8 || C == 16 || C == 32 || C == 64; }   // the channel counts fs2_resstack serves

// Stage i's operand format, and which of its ResBlock layers run as one fs2_resstack launch (window_walk, fs2_vocoder_resblock_runs)
static unsigned stage_tcv(const fs2_vocoder_model* m, int i) { return (m->f8_mask & (2 << i)) ? FS2_TC_VARIANT_F8 : 0; }
static bool stage_fused(const fs2_vocoder_model* m, int i) { return (m->fused_mask >> i) & 1; }
// A 128-channel stage pairs only with pair_mask bit 8 + i (its tiles are then packed at NB = 128, see fs2_vocoder_model::pair_mask)
static bool stage_pairs(const fs2_vocoder_model* m, int i, int C, int k) {
  const bool on = C == 128 ? (m->pair_mask >> (8 + i)) & 1 : ((m->pair_mask >> i) & 1) && resstack_width(C);
  return on && stage_tcv(m, i) && k <= m->pair_kmax;
}

// ------------------------------------------------------------------ ResBlock run planner (fs2_vocoder_resblock_runs)
// Cost of one fs2_resstack launch in ns per output row of the stage.  A work item computes MT * 128 slab rows for TILE output rows, and
// per slab row it spends `tap` ns per conv tap (the MMAs), `conv` ns per conv (the epilogue: operand split into shared memory, the
// barrier) and `run` ns per kernel size (x in through TMA and its split, the result out: the fp32 round trip of an intermediate
// between two runs is part of this term).  Fitted by least squares, by channels computed on chip, to the time of every cut of every
// ResBlock (scripts/resblock_runs_bench.py --candidates, B = 16 x 1012 frames, padded) on an H100 80GB HBM3 (SXM) at a 700 W power
// limit: V1's 64- and 32-channel stages (every cut within 2 % of the model) and V2's 16-channel stage (within 3 %).  The 8-channel
// stage, computed on chip as 16 channels, uses the 16-channel rates: they overestimate it by about 40 % but rank its cuts as measured.
struct RbNs { double tap, conv, run; };
static RbNs rb_ns(int Cm) {
  if (Cm >= 64) return {0.0169, 0.148, 0.215};
  if (Cm >= 32) return {0.0055, 0.063, 0.101};
  return {0.0026, 0.026, 0.041};
}

typedef fs2_resblock_run_t RbRun;
constexpr int RB_MAX_RUNS = (FS2_MAX_DIL + 4) * FS2_MAX_DIL;

// r.cost, H, TILE and slab of launching `a` (its j, d0, d1 are the caller's), or fs2_resstack's refusal of the shape
static int run_cost(const fs2_resstack_args& a, RbRun& r) {
  fs2_resstack_plan_t p;
  FS2_TRY(resstack_plan(&a, 1, p));
  const RbNs ns = rb_ns(a.C < 16 ? 16 : a.C);
  double per_slab_row = 0;
  for (int j = 0; j < a.n_kernels; j++) per_slab_row += ns.run + a.n_dil * 2 * (ns.conv + a.k[j] * ns.tap);
  r.H = p.H; r.TILE = p.TILE; r.slab = p.MT * 128;
  r.cost = per_slab_row * r.slab / r.TILE;
  return FS2_OK;
}

// The launches of stage i's ResBlocks (stage i in fused_mask): the whole group, or for each ResBlock the cut of its dilations into
// consecutive runs with the least modelled cost, whichever costs less (ties: fewer launches).  Returns the count.
static int stage_runs(const fs2_vocoder_model* m, int i, RbRun* out) {
  if (!resstack_width(m->c0 >> (i + 1))) return FS2_ERR_UNSUPPORTED;   // fused_mask serves 8 to 64 channels (128: pair_mask bit 8 + i)
  const fs2_resstack_args g = resblock_args(m, i, 1, 1, m->c0 >> (i + 1), nullptr, 1);
  RbRun whole{-1, 0, m->n_dil, 0, 0, 0, 0};
  const bool whole_ok = run_cost(g, whole) == FS2_OK;
  int n = 0;
  double split = 0;
  for (int j = 0; j < m->n_kernels; j++) {
    RbRun best[FS2_MAX_DIL];
    int nbest = 0;
    double best_cost = 0;
    for (int cuts = 0; cuts < 1 << (m->n_dil - 1); cuts++) {   // bit d: a run ends after dilation d
      RbRun cand[FS2_MAX_DIL];
      int nc = 0;
      double c = 0;
      bool ok = true;
      for (int d0 = 0; d0 < m->n_dil && ok;) {
        int d1 = d0 + 1;
        while (d1 < m->n_dil && !((cuts >> (d1 - 1)) & 1)) d1++;
        fs2_resstack_args a = resblock_run(g, j, d0, d1);
        a.accumulate = d1 == m->n_dil && j > 0;
        cand[nc] = RbRun{j, d0, d1, 0, 0, 0, 0};
        ok = run_cost(a, cand[nc]) == FS2_OK;
        c += cand[nc++].cost;
        d0 = d1;
      }
      if (ok && (!nbest || c < best_cost || (c == best_cost && nc < nbest))) {
        for (int r = 0; r < nc; r++) best[r] = cand[r];
        nbest = nc; best_cost = c;
      }
    }
    if (!nbest) {
      if (!whole_ok) return FS2_ERR_UNSUPPORTED;
      split = -1;
      break;
    }
    for (int r = 0; r < nbest; r++) out[n++] = best[r];
    split += best_cost;
  }
  if (whole_ok && (split < 0 || whole.cost <= split)) {
    out[0] = whole;
    return 1;
  }
  return n;
}

// ------------------------------------------------------------------ vocoder (fs2_vocoder_forward, _forward_window, _forward_streams)
// A window [f0, f1) is walked backward from its output samples to the rows every layer must compute (each conv: its consumers' rows
// widened by its radius, clipped to the utterance's logical extent), then forward in launch order, every layer computing only those
// rows with the kernels and arithmetic of the whole batch.  One walk makes both the plan (fs2_vocoder_window_plan) and, given a
// WinExec, the launches, so the two cannot disagree.  It issues two modes: fs2_vocoder_forward is the window [0, T) of a T-frame batch
// (every range is then [0, T * scale), every buffer [B][T * scale][C], and the walk runs the offline entry points), and the windowed
// calls run the unclipped plan of [0, frames) with every utterance at its own origin (OriginWindow).

struct Rows {
  int lo, hi;
  int n() const { return hi - lo; }
};
// [lo - by, hi + by) clipped to [0, cap); cap < 0: unclipped (the workspace bound of a window of hi - lo frames)
static Rows widen(Rows r, int by, long long cap) {
  r.lo -= by; r.hi += by;
  if (cap >= 0) { r.lo = r.lo > 0 ? r.lo : 0; r.hi = (long long)r.hi < cap ? r.hi : (int)cap; }
  return r;
}
static int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
static int pair_reach(const fs2_vocoder_model* m, int j, int d) { return (m->rb_k[j] - 1) * m->rb_dil[j][d] / 2 + (m->rb_k[j] - 1) / 2; }
// rows per mel frame at stage i's input, prod(rates[0, i)); i = n_stages: waveform samples per mel frame
static long long frame_rows(const fs2_vocoder_model* m, int i) {
  long long r = 1;
  for (int k = 0; k < i; k++) r *= m->rates[k];
  return r;
}

// A window buffer: logical rows [lo, lo + rows) of C floats each, utterances `rows` rows apart.
struct View {
  float* p; int lo, rows, C;
  // logical row 0 of utterance 0: the kernels address logical rows, and never dereference one outside [lo, lo + rows)
  float* at() const { return reinterpret_cast<float*>(reinterpret_cast<uintptr_t>(p) - (uintptr_t)lo * C * sizeof(float)); }
  int64_t bs() const { return (int64_t)rows * C; }
};

// What a walk issues: the batch's mel view and lengths, the waveform, and five buffers, each B * width floats (window_plan).
// org: NULL (the offline forward), or the windowed mode: the walk is then the unclipped plan of [0, frames), its rows are window rows,
// utterance b's window starts at its frame org[b] (origin_rows), and the mel is the staged window buffer.  pre_tc: conv_pre's
// tensor-core weights, or NULL where the caller's mel layout keeps conv_pre on the fp32 kernel.  table (windowed mode only): the
// multi-generator mode's generators and staged table (models NULL outside it); the walk plans and checks on m, generator 0.
struct WinExec {
  int B; cudaStream_t s;
  const float* mel; int64_t mel_bs, mel_rs;
  const int32_t* lens; const int32_t* org;
  const float* pre_tc;
  float* wav; int64_t wav_bs;
  float *bx, *bu, *bt, *r1, *r2;
  ModelTable table;
};

// fs2_conv1d arguments of a windowed launch: `cap` (a.T) is the layer's full logical length; residual off, as conv_args leaves it
static fs2_conv1d_args win_conv_args(const float* x, int64_t xbs, int64_t xrs, int B, int cap, int Cin, const View& y, int N, int taps) {
  fs2_conv1d_args c = conv_args(x, B, cap, Cin, N, taps, y.at());
  c.x_batch_stride = xbs; c.x_row_stride = xrs;
  c.y_batch_stride = y.bs(); c.y_row_stride = y.C;
  c.res_batch_stride = c.res_row_stride = 0;
  return c;
}

// The launches of window [f0, f1) of a T-frame batch (f1 <= T), appended to L in issue order; with ex, also issued.  T < 0: the plan of
// an unclipped [f0, f1) (no launches), whose row counts bound those of every window of f1 - f0 frames.  Refuses a model it cannot run
// before its first launch.
static int window_walk(const fs2_vocoder_model* m, int T, int f0, int f1, std::vector<fs2_vocoder_window_launch_t>& L, const WinExec* ex) {
  const int n = m->n_stages;
  int sc[FS2_MAX_STAGES + 1];                          // rows per mel frame at stage i's input (sc[n]: the waveform)
  for (int i = 0; i <= n; i++) sc[i] = (int)frame_rows(m, i);
  for (int i = 0; i < n; i++) {
    if (m->up_k[i] != 2 * m->rates[i] || (m->rates[i] & 1)) return FS2_ERR_UNSUPPORTED;
    if (stage_fused(m, i) && !stage_tcv(m, i)) return FS2_ERR_ARG;
  }
  auto cap = [&](int scale) { return T < 0 ? -1LL : (long long)T * scale; };
  // the kernels' logical length at `scale` rows per frame, and a launch's window: the windowed mode bounds every utterance by itself
  // (origin_rows); the offline forward passes no window, so it runs the offline entry points
  const int* org = ex ? ex->org : nullptr;
  auto len = [&](int scale) { return org ? ORIGIN_CAP : T * scale; };
  OriginWindow ow{};
  auto win = [&](const RowWindow& w) -> const OriginWindow* {
    ow = OriginWindow{w, org};
    return org ? &ow : nullptr;
  };
  // the launch's weights as fields of fs2_vocoder_model, which the multi-generator mode reads per work item
  LaunchWeights lw{};
  const ModelTable table = ex ? ex->table : ModelTable{};
  auto weights = [&](FieldRef w, FieldRef wt, FieldRef bias, int rb = 0, int d0 = 0) -> const LaunchWeights* {
    lw = LaunchWeights{table, w, wt, bias, rb, d0};
    return table.models ? &lw : nullptr;
  };
  auto ref = [&](const void* field, int add = 0) { return field_ref(m, field, add); };
  // ---- backward: O[i + 1] = the rows stage i's output must hold (O[0]: conv_pre's), U[i] = its ResBlocks' input, Q[i] = the
  // ConvTranspose's phase-group rows
  Rows O[FS2_MAX_STAGES + 1], U[FS2_MAX_STAGES], Q[FS2_MAX_STAGES];
  const Rows post = widen(Rows{f0 * sc[n], f1 * sc[n]}, 0, cap(sc[n]));
  O[n] = widen(post, 3, cap(sc[n]));
  for (int i = n - 1; i >= 0; i--) {
    int reach = 0;                                     // the widest ResBlock's receptive radius
    for (int j = 0; j < m->n_kernels; j++) {
      int r = 0;
      for (int d = 0; d < m->n_dil; d++) r += pair_reach(m, j, d);
      reach = r > reach ? r : reach;
    }
    const int u = m->rates[i];
    U[i] = widen(O[i + 1], reach, cap(sc[i + 1]));
    Q[i] = Rows{floor_div(U[i].lo, u), -floor_div(-U[i].hi, u)};
    O[i] = widen(Q[i], 1, cap(sc[i]));
  }
  // ---- forward
  auto add = [&](int layer, int stage, int j, int d, int scale, Rows y, Rows x, int src, int res_src, double flops) {
    fs2_vocoder_window_launch_t l{};
    l.layer = layer; l.stage = stage; l.j = j; l.d = d; l.scale = scale;
    l.y0 = y.lo; l.y1 = y.hi; l.x0 = x.lo; l.x1 = x.hi; l.src = src; l.res_src = res_src; l.flops = flops;
    L.push_back(l);
    return (int)L.size() - 1;
  };
  const int B = ex ? ex->B : 0;
  const int32_t* lens = ex ? ex->lens : nullptr;
  cudaStream_t s = ex ? ex->s : nullptr;
  int C = m->c0;
  const Rows mel = widen(O[0], 3, cap(1));
  int last = add(FS2_VW_CONV_PRE, -1, -1, -1, 1, O[0], mel, -1, -1, 2.0 * O[0].n() * m->n_mel * 7 * C);
  View bx{ex ? ex->bx : nullptr, O[0].lo, O[0].n(), C};
  if (ex) {
    fs2_conv1d_args c = win_conv_args(ex->mel, ex->mel_bs, ex->mel_rs, B, len(1), m->n_mel, bx, C, 7);
    c.w = m->w_pre; c.w_tc = ex->pre_tc; c.bias = m->b_pre; c.tc_variant = (m->f8_mask & 1) ? FS2_TC_VARIANT_F8 : 0;
    c.x_lens = lens; c.lens_scale = 1;
    FS2_TRY(conv1d_dispatch(&c, s, win({O[0].lo, O[0].hi, mel.hi}), weights(ref(&m->w_pre), ref(&m->w_pre_tc), ref(&m->b_pre))));
  }
  const float inv_nk = 1.f / (float)m->n_kernels;
  for (int i = 0; i < n; i++) {
    const int u = m->rates[i], Co = C / 2, s0 = sc[i], s1 = sc[i + 1];
    const unsigned tcv = stage_tcv(m, i);
    // ---- lrelu + ConvTranspose1d as two 2-tap phase-group convolutions (hifigan/models.py:152-153): rows Q[i] of [u * Co] = the
    // next rate's rows [Q.lo * u, Q.hi * u)
    const double up_flops = 2.0 * Q[i].n() * C * 2 * (u / 2) * Co;
    const View bu{ex ? ex->bu : nullptr, Q[i].lo, Q[i].n(), u * Co};
    int up_src = -1;
    for (int g = 0; g < 2; g++) {
      const Rows x = widen(Rows{Q[i].lo - (g == 0), Q[i].hi + (g == 1)}, 0, cap(s0));
      up_src = add(g == 0 ? FS2_VW_UP_A : FS2_VW_UP_B, i, -1, -1, s0, Q[i], x, last, -1, up_flops);
      if (!ex) continue;
      const size_t off = (size_t)g * (u / 2) * Co;    // group g writes output channels [off, off + (u/2)*Co) of each [u*Co] row
      fs2_conv1d_args c = win_conv_args(bx.at(), bx.bs(), C, B, len(s0), C, bu, (u / 2) * Co, 2);
      c.y += off;
      c.pad_left = g == 0 ? 1 : 0;
      c.w = g == 0 ? m->w_up_a[i] : m->w_up_b[i];
      c.w_tc = g == 0 ? m->w_up_a_tc[i] : m->w_up_b_tc[i];
      c.bias = m->b_up[i] + off;
      c.in_act = FS2_ACT_LRELU; c.in_slope = 0.1f; c.tc_variant = tcv;
      c.x_lens = lens; c.lens_scale = s0;
      FS2_TRY(conv1d_dispatch(&c, s, win({Q[i].lo, Q[i].hi, x.hi}),
                              weights(ref(g == 0 ? &m->w_up_a[i] : &m->w_up_b[i]), ref(g == 0 ? &m->w_up_a_tc[i] : &m->w_up_b_tc[i]),
                                      ref(&m->b_up[i], (int)off))));
    }
    C = Co;
    const View in{bu.p, bu.lo * u, bu.rows * u, C};    // the same buffer at the ResBlocks' rate
    const long long cap1 = cap(s1);
    bx = View{bx.p, O[i + 1].lo, O[i + 1].n(), C};
    // ---- mean of the multi-receptive-field ResBlocks (models.py:154-160, ResBlock.forward :96-103).  Its launches: in a fused stage
    // the planner's runs (fs2_vocoder_resblock_runs), each widened by its total reach; else one (j, d, d + 1) per layer, a fused pair
    // (the intermediate stays on chip) or the two convs through bt.
    const bool fused = stage_fused(m, i);
    RbRun runs[RB_MAX_RUNS];
    int nr = 0;
    if (fused) {
      nr = stage_runs(m, i, runs);
      if (nr < 0) return nr;
    } else {
      for (int j = 0; j < m->n_kernels; j++)
        for (int d = 0; d < m->n_dil; d++) runs[nr++] = RbRun{j, d, d + 1, 0, 0, 0, 0};
    }
    const fs2_resstack_args group = ex ? resblock_args(m, i, B, len(s1), C, lens, s1) : fs2_resstack_args{};
    auto conv_flops = [&](Rows y, int k) { return 2.0 * y.n() * C * k * C; };
    View r = in;
    int r_src = up_src;
    for (int q = 0; q < nr; q++) {
      const RbRun& run = runs[q];
      const bool lastd = run.d1 == m->n_dil;          // the last layer of a ResBlock adds its share of the mean into bx
      if (run.d0 == 0) { r = in; r_src = up_src; }
      // R[d]: output rows of ResBlock j's pair d; the launch's FLOPs are its convs' over their rows
      Rows R[FS2_MAX_DIL], y = O[i + 1], x = U[i];
      double fl = 0;
      for (int j = run.j < 0 ? 0 : run.j; j < (run.j < 0 ? m->n_kernels : run.j + 1); j++) {
        const int k = m->rb_k[j];
        R[m->n_dil - 1] = O[i + 1];
        for (int d = m->n_dil - 1; d > 0; d--) R[d - 1] = widen(R[d], pair_reach(m, j, d), cap1);
        for (int d = run.d0; d < run.d1; d++) fl += conv_flops(widen(R[d], (k - 1) / 2, cap1), k) + conv_flops(R[d], k);
      }
      if (run.j >= 0) {
        y = R[run.d1 - 1];
        x = widen(R[run.d0], pair_reach(m, run.j, run.d0), cap1);
      }
      const View dst{lastd ? bx.p : (ex && r.p == ex->r1 ? ex->r2 : (ex ? ex->r1 : nullptr)), y.lo, y.n(), C};
      const float alpha = lastd ? inv_nk : 1.f;
      const int accumulate = lastd && run.j > 0;
      if (fused || stage_pairs(m, i, C, m->rb_k[run.j])) {
        r_src = add(fused ? FS2_VW_RB_GROUP : FS2_VW_RB_PAIR, i, run.j, run.j < 0 ? -1 : run.d0, s1, y, x, r_src, fused ? -1 : r_src, fl);
        if (ex) {
          fs2_resstack_args a = group;                 // the whole group: alpha 0 (the mean), no accumulate
          if (run.j >= 0) {
            a = resblock_run(group, run.j, run.d0, run.d1);
            a.alpha = alpha; a.accumulate = accumulate;
          }
          a.x = r.p; a.y = dst.p;
          FS2_TRY(resstack(&a, s, win({y.lo, y.hi, r.lo + r.rows}),
                           weights({}, {}, {}, i * m->n_kernels + (run.j < 0 ? 0 : run.j), run.j < 0 ? 0 : run.d0), r.lo, C == 128));
        }
      } else {
        const int j = run.j, d = run.d0, rb = i * m->n_kernels + j, k = m->rb_k[j];
        const Rows mid = widen(y, (k - 1) / 2, cap1);
        const int c1 = add(FS2_VW_RB_CONV1, i, j, d, s1, mid, x, r_src, -1, conv_flops(mid, k));
        r_src = add(FS2_VW_RB_CONV2, i, j, d, s1, y, mid, c1, r_src, conv_flops(y, k));
        if (ex) {
          const int dil = m->rb_dil[j][d];
          const View t{ex->bt, mid.lo, mid.n(), C};
          fs2_conv1d_args c = win_conv_args(r.at(), r.bs(), C, B, len(s1), C, t, C, k);
          c.w = m->w_rb1[rb][d]; c.w_tc = m->w_rb1_tc[rb][d]; c.bias = m->b_rb1[rb][d]; c.tc_variant = tcv;
          c.dilation = dil; c.pad_left = (k * dil - dil) / 2;
          c.in_act = c.out_act = FS2_ACT_LRELU; c.in_slope = c.out_slope = 0.1f;
          c.x_lens = lens; c.lens_scale = s1;
          FS2_TRY(conv1d_dispatch(&c, s, win({mid.lo, mid.hi, x.hi}), weights(ref(&m->w_rb1[rb][d]), ref(&m->w_rb1_tc[rb][d]), ref(&m->b_rb1[rb][d]))));
          c = win_conv_args(t.at(), t.bs(), C, B, len(s1), C, dst, C, k);
          c.w = m->w_rb2[rb][d]; c.w_tc = m->w_rb2_tc[rb][d]; c.bias = m->b_rb2[rb][d]; c.tc_variant = tcv;
          c.res = r.at(); c.res_batch_stride = r.bs(); c.res_row_stride = C;
          c.alpha = alpha; c.accumulate = accumulate;
          c.x_lens = lens; c.lens_scale = s1;
          FS2_TRY(conv1d_dispatch(&c, s, win({y.lo, y.hi, mid.hi}), weights(ref(&m->w_rb2[rb][d]), ref(&m->w_rb2_tc[rb][d]), ref(&m->b_rb2[rb][d]))));
        }
      }
      r = dst;
    }
    last = r_src;
  }
  add(FS2_VW_CONV_POST, -1, -1, -1, sc[n], post, O[n], last, -1, 2.0 * post.n() * C * 7);
  if (!ex) return FS2_OK;
  fs2_conv_post_args p{};
  p.x = bx.at(); p.B = B; p.T = len(sc[n]); p.C = C; p.w = m->w_post; p.bias = m->b_post; p.taps = 7; p.in_slope = 0.01f;
  p.wav = ex->wav - post.lo;                           // sample f0 * up is the caller's wav[0]
  p.lens = lens; p.lens_scale = sc[n];
  return conv_post(&p, s, win({post.lo, post.hi, O[n].hi}), weights(ref(&m->w_post), {}, ref(&m->b_post)), bx.bs(),
                   ex->wav_bs);   // offline: the strides are its defaults
}

// The plan of [0, frames) clipped at T (T < 0: unclipped, the bound of every window of `frames` frames), and the floats per utterance
// of each of the five buffers that hold it: the widest output of its launches
static int window_plan(const fs2_vocoder_model* m, int T, int frames, std::vector<fs2_vocoder_window_launch_t>& L, size_t& width) {
  FS2_TRY(window_walk(m, T, 0, frames, L, nullptr));
  width = 0;
  for (const auto& l : L) {
    size_t ch = 0;                                     // floats per output row
    if (l.layer == FS2_VW_CONV_PRE) ch = (size_t)m->c0;
    else if (l.layer == FS2_VW_UP_A || l.layer == FS2_VW_UP_B) ch = (size_t)m->rates[l.stage] * (m->c0 >> (l.stage + 1));
    else if (l.layer != FS2_VW_CONV_POST) ch = (size_t)(m->c0 >> (l.stage + 1));
    const size_t w = (size_t)(l.y1 - l.y0) * ch;
    width = w > width ? w : width;
  }
  return FS2_OK;
}

// fs2_vocoder_forward: the window [0, T) of the batch, on buffers of B * T * max(c0, max_i prod(rates[0, i]) * c_i) floats
static int vocoder_forward_impl(const fs2_vocoder_model* m, const fs2_vocoder_args* a, cudaStream_t s, Arena& ar) {
  std::vector<fs2_vocoder_window_launch_t> L;
  size_t width = 0;
  FS2_TRY(window_plan(m, a->T, a->T, L, width));
  const size_t nf = (size_t)a->B * width;
  WinExec ex{a->B, s, a->mel, a->mel_batch_stride, a->mel_row_stride, a->mel_lens, nullptr, m->w_pre_tc, a->wav,
             a->T * frame_rows(m, m->n_stages), ar.f32(nf), ar.f32(nf), ar.f32(nf), ar.f32(nf), ar.f32(nf)};
  if (ar.dry) return FS2_OK;
  if (!ex.bx || !ex.bu || !ex.bt || !ex.r1 || !ex.r2) return FS2_ERR_WORKSPACE;
  L.clear();
  return window_walk(m, a->T, 0, a->T, L, &ex);
}

// fs2_vocoder_forward_window and _streams: the unclipped plan of [0, frames) once for the whole batch, each stream at its own origin.
// The mel cone (conv_pre's input rows [x0, x1) of that plan) is staged first, [B][x1 - x0][n_mel], with the streams' origins and
// lengths, so that conv_pre reads one batch-strided buffer and every launch the same two tables whichever call passed them.
// mg (gen set): the multi-generator mode, whose staged generator table is a third one.
struct MultiGen { const fs2_vocoder_model* models_dev; const int32_t* gen; int n; };
static int vocoder_windowed_impl(const fs2_vocoder_model* m, const MelSource& src, int B, int frames, float* wav, int64_t wav_bs,
                                 const float* pre_tc, cudaStream_t s, Arena& ar, const MultiGen& mg = MultiGen{}) {
  std::vector<fs2_vocoder_window_launch_t> L;
  size_t width = 0;
  FS2_TRY(window_plan(m, -1, frames, L, width));
  const int x0 = L[0].x0, rows = L[0].x1 - L[0].x0;     // launch 0 is conv_pre
  const size_t nf = (size_t)B * width;
  float* mel = ar.f32((size_t)B * rows * m->n_mel);
  int32_t* org = (int32_t*)ar.take((size_t)B * sizeof(int32_t));
  int32_t* lens = (int32_t*)ar.take((size_t)B * sizeof(int32_t));
  int32_t* gen = mg.gen ? (int32_t*)ar.take((size_t)B * sizeof(int32_t)) : nullptr;
  WinExec ex{B, s, nullptr, (int64_t)rows * m->n_mel, m->n_mel, lens, org, pre_tc, wav, wav_bs,
             ar.f32(nf), ar.f32(nf), ar.f32(nf), ar.f32(nf), ar.f32(nf), model_table(mg.gen ? mg.models_dev : nullptr, gen)};
  if (ar.dry) return FS2_OK;
  if (!mel || !org || !lens || (mg.gen && !gen) || !ex.bx || !ex.bu || !ex.bt || !ex.r1 || !ex.r2) return FS2_ERR_WORKSPACE;
  FS2_TRY(stage_mel(src, B, x0, rows, m->n_mel, mel, org, lens, mg.gen, mg.n, gen, s));
  ex.mel = mel - (ptrdiff_t)x0 * m->n_mel;             // window row 0 of stream 0 (the conv reads rows [x0, x1) only)
  L.clear();
  return window_walk(m, -1, 0, frames, L, &ex);
}

}  // namespace fs2

// ====================================================================== extern "C"
using namespace fs2;
#define S(x) ((cudaStream_t)(x))

extern "C" {

int fs2_abi_version(void) { return 12; }
int fs2_conv_tc_block(int N) { return conv_tc_nb(N, 128); }
int fs2_conv_tc_block_f8(int N) { return conv_tc_nb(N, 64); }
int fs2_conv_tc_plan(const fs2_conv1d_args* a, int num_sms, fs2_conv_tc_plan_t* out) { return conv_tc_plan_query(a, num_sms, out); }
int fs2_conv_simt_plan(const fs2_conv1d_args* a, int num_sms, fs2_conv_simt_plan_t* out) { return conv_simt_plan(a, num_sms, out); }
int64_t fs2_kernel_launch_count(void) { return (int64_t)g_launch_count.load(); }
// fs2_control_args is not in the fs2_struct_size table (its indices are pinned at 0..18): its layout is pinned here and in the binding
static_assert(sizeof(fs2_control_args) == 48, "fs2_control_args: two pointers and four int64 strides");
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
    case 16: return sizeof(fs2_conv_tc_plan_t);
    case 17: return sizeof(fs2_conv_simt_plan_t);
    case 18: return sizeof(fs2_resstack_plan_t);
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
int fs2_resstack_plan(const fs2_resstack_args* a, int num_sms, fs2_resstack_plan_t* out) { return out ? resstack_plan(a, num_sms, *out) : FS2_ERR_ARG; }
int fs2_add_positions(float* x, const float* pos, int B, int T, int D, fs2_stream_t st) { return add_positions(x, pos, B, T, D, S(st)); }
int fs2_transpose_bct_to_btc(const float* in, float* out, int B, int C, int T, fs2_stream_t st) {
  return transpose_bct_to_btc(in, out, B, C, T, S(st));
}

size_t fs2_encode_workspace_bytes(const fs2_acoustic_model* m, int B, int L) {
  if (!model_ok(m) || B <= 0 || L <= 0) return 0;
  Arena ar(nullptr, 0);
  fs2_encode_args a{};
  a.B = B; a.L = L;
  encode_impl(m, &a, nullptr, nullptr, ar, false);
  return ar.off + 256;
}

static bool control_ok(const fs2_control_args* c, int ragged) {
  return (ragged == 0 || ragged == 1) &&
         (!c || (c->p_stride_b >= 0 && c->p_stride_l >= 0 && c->d_stride_b >= 0 && c->d_stride_l >= 0));
}

// voices: NULL, or the voices mode (m = voices->models[0], checked by the caller)
static int encode_call(const fs2_acoustic_model* m, const fs2_encode_args* a, const fs2_control_args* ctl, int ragged, fs2_stream_t st,
                       const fs2_acoustic_voices* voices = nullptr) {
  if (!model_ok(m) || !a || a->B <= 0 || a->L <= 0 || !control_ok(ctl, ragged)) return FS2_ERR_ARG;
  if (!a->texts || !a->src_lens || !a->logd_pred || !a->mel_lens || !a->cum_dur || !a->x_adapted ||
      !a->len_stats || !a->workspace)
    return FS2_ERR_ARG;
  if (!a->d_target && !a->d_rounded) return FS2_ERR_ARG;
  if (m->d_model / m->n_head != 128) return FS2_ERR_UNSUPPORTED;
  Arena ar(a->workspace, a->workspace_bytes);
  return encode_impl(m, a, ctl, S(st), ar, ragged != 0, voices);
}
int fs2_acoustic_encode_ctl(const fs2_acoustic_model* m, const fs2_encode_args* a, const fs2_control_args* ctl, int ragged, fs2_stream_t st) {
  return encode_call(m, a, ctl, ragged, st);
}
int fs2_acoustic_encode(const fs2_acoustic_model* m, const fs2_encode_args* a, fs2_stream_t st) { return fs2_acoustic_encode_ctl(m, a, nullptr, 0, st); }
int fs2_acoustic_encode_ragged(const fs2_acoustic_model* m, const fs2_encode_args* a, fs2_stream_t st) { return fs2_acoustic_encode_ctl(m, a, nullptr, 1, st); }

size_t fs2_decode_workspace_bytes(const fs2_acoustic_model* m, int B, int T) {
  if (!model_ok(m) || B <= 0 || T <= 0) return 0;
  Arena ar(nullptr, 0);
  fs2_decode_args a{};
  a.B = B; a.T = T;
  decode_impl(m, &a, nullptr, nullptr, ar, false);
  return ar.off + 256;
}

static int decode_call(const fs2_acoustic_model* m, const fs2_decode_args* a, const fs2_control_args* ctl, int ragged, fs2_stream_t st,
                       const fs2_acoustic_voices* voices = nullptr) {
  if (!model_ok(m) || !a || a->B <= 0 || a->L <= 0 || a->T <= 0 || !control_ok(ctl, ragged)) return FS2_ERR_ARG;
  if (!a->x_adapted || !a->cum_dur || !a->mel_mask_lens || !a->mel || !a->postnet_mel || !a->workspace) return FS2_ERR_ARG;
  if (m->d_model / m->n_head != 128) return FS2_ERR_UNSUPPORTED;
  Arena ar(a->workspace, a->workspace_bytes);
  return decode_impl(m, a, ctl, S(st), ar, ragged != 0, voices);
}
int fs2_acoustic_decode_ctl(const fs2_acoustic_model* m, const fs2_decode_args* a, const fs2_control_args* ctl, int ragged, fs2_stream_t st) {
  return decode_call(m, a, ctl, ragged, st);
}
int fs2_acoustic_decode(const fs2_acoustic_model* m, const fs2_decode_args* a, fs2_stream_t st) { return fs2_acoustic_decode_ctl(m, a, nullptr, 0, st); }
int fs2_acoustic_decode_ragged(const fs2_acoustic_model* m, const fs2_decode_args* a, fs2_stream_t st) { return fs2_acoustic_decode_ctl(m, a, nullptr, 1, st); }

static_assert(sizeof(fs2_acoustic_voices) == 32, "fs2_acoustic_voices: an int32 and three pointers");

// Model k of a table call (voices, generators) runs on model 0's plan and kernels, so each of its weight pointers q must be NULL where
// model 0's p is, else at the same address modulo 16 (the format choices and alignment checks made on model 0).
static bool same_ptr(const float* p, const float* q) { return !p == !q && ((uintptr_t)p & 15u) == ((uintptr_t)q & 15u); }

// Voice k of a voices call: the same config and precision policy as voice 0, and its pointers as same_ptr asks.
static bool same_acoustic_layout(const fs2_acoustic_model* a, const fs2_acoustic_model* b) {
  if (a->d_model != b->d_model || a->n_head != b->n_head || a->d_inner != b->d_inner || a->k1 != b->k1 || a->k2 != b->k2 ||
      a->n_enc != b->n_enc || a->n_dec != b->n_dec || a->n_mel != b->n_mel || a->vp_filter != b->vp_filter ||
      a->vp_kernel != b->vp_kernel || a->n_bins != b->n_bins || a->n_vocab != b->n_vocab || a->n_speakers != b->n_speakers ||
      a->tc_mask != b->tc_mask || a->pitch_frame_level != b->pitch_frame_level || a->energy_frame_level != b->energy_frame_level ||
      a->n_postnet != b->n_postnet || a->post_k != b->post_k)
    return false;
  for (int i = 0; i < a->n_postnet; i++)
    if (a->post_cin[i] != b->post_cin[i] || a->post_cout[i] != b->post_cout[i]) return false;
  // the weight structs hold pointers only: compared as arrays of them
  auto same_all = [](const void* p, const void* q, size_t bytes) {
    bool ok = true;
    for (size_t i = 0; i < bytes / sizeof(const float*); i++) ok = ok && same_ptr(((const float* const*)p)[i], ((const float* const*)q)[i]);
    return ok;
  };
  bool ok = same_ptr(a->word_emb, b->word_emb) && same_ptr(a->enc_pos, b->enc_pos) && same_ptr(a->dec_pos, b->dec_pos) &&
            same_ptr(a->spk_emb, b->spk_emb) && same_ptr(a->pitch_bins, b->pitch_bins) && same_ptr(a->energy_bins, b->energy_bins) &&
            same_ptr(a->pitch_emb, b->pitch_emb) && same_ptr(a->energy_emb, b->energy_emb) && same_ptr(a->w_mel, b->w_mel) &&
            same_ptr(a->b_mel, b->b_mel) && same_ptr(a->w_mel_tc, b->w_mel_tc);
  for (int i = 0; i < a->n_enc; i++) ok = ok && same_all(&a->enc[i], &b->enc[i], sizeof(fs2_fft_block_weights));
  for (int i = 0; i < a->n_dec; i++) ok = ok && same_all(&a->dec[i], &b->dec[i], sizeof(fs2_fft_block_weights));
  ok = ok && same_all(&a->dur, &b->dur, sizeof(fs2_predictor_weights)) && same_all(&a->pitch, &b->pitch, sizeof(fs2_predictor_weights)) &&
       same_all(&a->energy, &b->energy, sizeof(fs2_predictor_weights));
  for (int i = 0; i < a->n_postnet; i++)
    ok = ok && same_ptr(a->w_post[i], b->w_post[i]) && same_ptr(a->b_post[i], b->b_post[i]) && same_ptr(a->w_post_tc[i], b->w_post_tc[i]);
  return ok;
}

// n, the models and their layouts (what the workspace bounds need); calls also need models_dev and voice
static bool voice_models_ok(const fs2_acoustic_voices* v) {
  if (!v || v->n < 1 || v->n > FS2_MAX_VOICES || !v->models) return false;
  for (int k = 0; k < v->n; k++)
    if (!model_ok(v->models[k]) || !same_acoustic_layout(v->models[0], v->models[k])) return false;
  return true;
}

size_t fs2_encode_voices_workspace_bytes(const fs2_acoustic_voices* v, int B, int L) {
  if (!voice_models_ok(v) || B <= 0 || L <= 0) return 0;
  Arena ar(nullptr, 0);
  fs2_encode_args a{};
  a.B = B; a.L = L;
  encode_impl(v->models[0], &a, nullptr, nullptr, ar, false, v);
  return ar.off + 256;
}

size_t fs2_decode_voices_workspace_bytes(const fs2_acoustic_voices* v, int B, int T) {
  if (!voice_models_ok(v) || B <= 0 || T <= 0) return 0;
  Arena ar(nullptr, 0);
  fs2_decode_args a{};
  a.B = B; a.T = T;
  decode_impl(v->models[0], &a, nullptr, nullptr, ar, false, v);
  return ar.off + 256;
}

int fs2_acoustic_encode_voices(const fs2_acoustic_voices* v, const fs2_encode_args* a, const fs2_control_args* ctl, int ragged,
                               fs2_stream_t st) {
  if (!voice_models_ok(v) || !v->models_dev || !v->voice || !a) return FS2_ERR_ARG;
  for (int k = 0; k < v->n; k++)
    if (a->L > v->models[k]->enc_pos_rows) return FS2_ERR_ARG;
  return encode_call(v->models[0], a, ctl, ragged, st, v);
}

int fs2_acoustic_decode_voices(const fs2_acoustic_voices* v, const fs2_decode_args* a, const fs2_control_args* ctl, int ragged,
                               fs2_stream_t st) {
  if (!voice_models_ok(v) || !v->models_dev || !v->voice || !a) return FS2_ERR_ARG;
  for (int k = 0; k < v->n; k++)
    if (a->T > v->models[k]->dec_pos_rows) return FS2_ERR_ARG;
  return decode_call(v->models[0], a, ctl, ragged, st, v);
}

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
  if (vocoder_forward_impl(m, &a, nullptr, ar) != FS2_OK) return 0;
  return ar.off + 256;
}

int fs2_vocoder_forward(const fs2_vocoder_model* m, const fs2_vocoder_args* a, fs2_stream_t st) {
  if (!vocoder_ok(m) || !a || a->B <= 0 || a->T <= 0 || !a->mel || !a->wav || !a->workspace) return FS2_ERR_ARG;
  Arena ar(a->workspace, a->workspace_bytes);
  return vocoder_forward_impl(m, a, S(st), ar);
}

// fs2_vocoder_window_args and fs2_vocoder_window_launch_t are not in the fs2_struct_size table (it stays at 0..18): pinned here and in
// the binding
static_assert(sizeof(fs2_vocoder_window_args) == 80, "fs2_vocoder_window_args: fs2_vocoder_args' fields, f0, f1, wav_batch_stride");
static_assert(sizeof(fs2_vocoder_window_launch_t) == 56, "fs2_vocoder_window_launch_t: twelve int32 and a double");

// Row counts of a window must fit the kernels' int rows with the halo: frames (and T) times prod(rates) below 2^30
static bool window_rows_ok(const fs2_vocoder_model* m, long long frames) { return frames * frame_rows(m, m->n_stages) < (1LL << 30); }

size_t fs2_vocoder_streams_workspace_bytes(const fs2_vocoder_model* m, int B, int frames) {
  if (!vocoder_ok(m) || B <= 0 || frames <= 0 || !window_rows_ok(m, frames)) return 0;
  Arena ar(nullptr, 0);
  if (vocoder_windowed_impl(m, MelSource{}, B, frames, nullptr, 0, nullptr, nullptr, ar) != FS2_OK) return 0;
  return ar.off + 256;
}

size_t fs2_vocoder_window_workspace_bytes(const fs2_vocoder_model* m, int B, int frames) {
  return fs2_vocoder_streams_workspace_bytes(m, B, frames);
}

int fs2_vocoder_forward_window(const fs2_vocoder_model* m, const fs2_vocoder_window_args* a, fs2_stream_t st) {
  if (!vocoder_ok(m) || !a || a->B <= 0 || a->T <= 0 || !a->mel || !a->wav || !a->workspace) return FS2_ERR_ARG;
  if (a->f0 < 0 || a->f1 <= a->f0 || a->f0 >= a->T || !window_rows_ok(m, a->T)) return FS2_ERR_ARG;
  const int frames = (a->f1 < a->T ? a->f1 : a->T) - a->f0;
  if (a->B > 1 && a->wav_batch_stride < frames * frame_rows(m, m->n_stages)) return FS2_ERR_ARG;
  // every stream starts at f0 and has clamp(mel_lens[b], 0, T) frames (T without mel_lens): the kernels read no row at or past T
  const MelSource src{nullptr, a->mel, a->mel_batch_stride, a->mel_row_stride, nullptr, a->f0, a->mel_lens, a->T};
  // conv_pre runs on the backend the caller's mel layout selects, as fs2_vocoder_forward's does on the same mel
  fs2_conv1d_args pre = conv_args(a->mel, a->B, a->T, m->n_mel, m->c0, 7, nullptr);
  pre.x_batch_stride = a->mel_batch_stride; pre.x_row_stride = a->mel_row_stride;
  Arena ar(a->workspace, a->workspace_bytes);
  return vocoder_windowed_impl(m, src, a->B, frames, a->wav, a->wav_batch_stride, conv_tc_supported(&pre) ? m->w_pre_tc : nullptr, S(st),
                               ar);
}

static_assert(sizeof(fs2_vocoder_streams_args) == 64, "fs2_vocoder_streams_args: two int32, five pointers, an int64 and a size_t");

// The streams call, its mel rows addressed as rings of ring[b] rows when ring is set (fs2_vocoder_forward_streams_ring)
static int vocoder_streams(const fs2_vocoder_model* m, const fs2_vocoder_streams_args* a, const int32_t* ring, fs2_stream_t st) {
  if (!vocoder_ok(m) || !a || a->B <= 0 || a->frames <= 0 || !window_rows_ok(m, a->frames)) return FS2_ERR_ARG;
  if (!a->mel || !a->mel_lens || !a->f0 || !a->wav || !a->workspace) return FS2_ERR_ARG;
  if (a->B > 1 && a->wav_batch_stride < a->frames * frame_rows(m, m->n_stages)) return FS2_ERR_ARG;
  if (a->workspace_bytes < fs2_vocoder_streams_workspace_bytes(m, a->B, a->frames)) return FS2_ERR_ARG;
  const MelSource src{a->mel, nullptr, 0, 0, a->f0, 0, a->mel_lens, INT32_MAX, ring};
  Arena ar(a->workspace, a->workspace_bytes);
  return vocoder_windowed_impl(m, src, a->B, a->frames, a->wav, a->wav_batch_stride, m->w_pre_tc, S(st), ar);
}

int fs2_vocoder_forward_streams(const fs2_vocoder_model* m, const fs2_vocoder_streams_args* a, fs2_stream_t st) {
  return vocoder_streams(m, a, nullptr, st);
}

static_assert(sizeof(fs2_vocoder_streams_ring_args) == 72, "fs2_vocoder_streams_ring_args: fs2_vocoder_streams_args' fields and cap");
static_assert(sizeof(fs2_mel_ring_record_t) == 56, "fs2_mel_ring_record_t: a pointer, three int64, a pointer, an int64, two int32");
static_assert(sizeof(fs2_mel_ring_append_args) == 24, "fs2_mel_ring_append_args: a pointer and three int32");

int fs2_vocoder_forward_streams_ring(const fs2_vocoder_model* m, const fs2_vocoder_streams_ring_args* a, fs2_stream_t st) {
  if (!a || !a->cap) return FS2_ERR_ARG;
  const fs2_vocoder_streams_args s{a->B, a->frames, a->mel, a->mel_lens, a->f0, a->wav, a->wav_batch_stride, a->workspace,
                                   a->workspace_bytes};
  return vocoder_streams(m, &s, a->cap, st);
}

int fs2_mel_ring_append(const fs2_mel_ring_append_args* a, fs2_stream_t st) { return mel_ring_append(a, S(st)); }

static_assert(sizeof(fs2_vocoder_streams_multi_args) == 88,
              "fs2_vocoder_streams_multi_args: fs2_vocoder_streams_ring_args' fields, gen and models_dev");

// Generator k of a multi-generator call: the same architecture and masks as generator 0, and its pointers as same_ptr asks.
static bool same_generator_layout(const fs2_vocoder_model* a, const fs2_vocoder_model* b) {
  if (a->n_mel != b->n_mel || a->c0 != b->c0 || a->n_stages != b->n_stages || a->n_kernels != b->n_kernels || a->n_dil != b->n_dil ||
      a->f8_mask != b->f8_mask || a->fused_mask != b->fused_mask || a->pair_mask != b->pair_mask || a->pair_kmax != b->pair_kmax)
    return false;
  for (int i = 0; i < a->n_stages; i++)
    if (a->rates[i] != b->rates[i] || a->up_k[i] != b->up_k[i]) return false;
  for (int j = 0; j < a->n_kernels; j++) {
    if (a->rb_k[j] != b->rb_k[j]) return false;
    for (int d = 0; d < a->n_dil; d++)
      if (a->rb_dil[j][d] != b->rb_dil[j][d]) return false;
  }
  bool ok = same_ptr(a->w_pre, b->w_pre) && same_ptr(a->b_pre, b->b_pre) && same_ptr(a->w_post, b->w_post) && same_ptr(a->b_post, b->b_post) &&
            same_ptr(a->w_pre_tc, b->w_pre_tc);
  for (int i = 0; i < a->n_stages; i++)
    ok = ok && same_ptr(a->w_up_a[i], b->w_up_a[i]) && same_ptr(a->w_up_b[i], b->w_up_b[i]) && same_ptr(a->b_up[i], b->b_up[i]) &&
         same_ptr(a->w_up_a_tc[i], b->w_up_a_tc[i]) && same_ptr(a->w_up_b_tc[i], b->w_up_b_tc[i]);
  for (int rb = 0; rb < a->n_stages * a->n_kernels; rb++)
    for (int d = 0; d < a->n_dil; d++)
      ok = ok && same_ptr(a->w_rb1[rb][d], b->w_rb1[rb][d]) && same_ptr(a->b_rb1[rb][d], b->b_rb1[rb][d]) && same_ptr(a->w_rb2[rb][d], b->w_rb2[rb][d]) &&
           same_ptr(a->b_rb2[rb][d], b->b_rb2[rb][d]) && same_ptr(a->w_rb1_tc[rb][d], b->w_rb1_tc[rb][d]) && same_ptr(a->w_rb2_tc[rb][d], b->w_rb2_tc[rb][d]);
  return ok;
}

static bool generators_ok(const fs2_vocoder_model* const* models, int n_models) {
  if (!models || n_models < 1 || n_models > FS2_MAX_GENERATORS) return false;
  for (int k = 0; k < n_models; k++)
    if (!vocoder_ok(models[k]) || !same_generator_layout(models[0], models[k])) return false;
  return true;
}

size_t fs2_vocoder_streams_multi_workspace_bytes(const fs2_vocoder_model* const* models, int n_models, int B, int frames) {
  if (!generators_ok(models, n_models) || B <= 0 || frames <= 0 || !window_rows_ok(models[0], frames)) return 0;
  Arena ar(nullptr, 0);
  const MultiGen dry{nullptr, reinterpret_cast<const int32_t*>(16), n_models};   // a dry run counts the generator table's bytes only
  if (vocoder_windowed_impl(models[0], MelSource{}, B, frames, nullptr, 0, nullptr, nullptr, ar, dry) != FS2_OK) return 0;
  return ar.off + 256;
}

int fs2_vocoder_forward_streams_multi(const fs2_vocoder_model* const* models, int n_models, const fs2_vocoder_streams_multi_args* a,
                                      fs2_stream_t st) {
  if (!generators_ok(models, n_models) || !a || !a->gen || !a->models_dev) return FS2_ERR_ARG;
  const fs2_vocoder_model* m = models[0];
  if (a->B <= 0 || a->frames <= 0 || !window_rows_ok(m, a->frames)) return FS2_ERR_ARG;
  if (!a->mel || !a->mel_lens || !a->f0 || !a->wav || !a->workspace) return FS2_ERR_ARG;
  if (a->B > 1 && a->wav_batch_stride < a->frames * frame_rows(m, m->n_stages)) return FS2_ERR_ARG;
  if (a->workspace_bytes < fs2_vocoder_streams_multi_workspace_bytes(models, n_models, a->B, a->frames)) return FS2_ERR_ARG;
  const MelSource src{a->mel, nullptr, 0, 0, a->f0, 0, a->mel_lens, INT32_MAX, a->cap};
  Arena ar(a->workspace, a->workspace_bytes);
  return vocoder_windowed_impl(m, src, a->B, a->frames, a->wav, a->wav_batch_stride, m->w_pre_tc, S(st), ar,
                               MultiGen{a->models_dev, a->gen, n_models});
}

static_assert(sizeof(fs2_resblock_run_t) == 32, "fs2_resblock_run_t: six int32 and a double");

int fs2_vocoder_resblock_runs(const fs2_vocoder_model* m, int stage, fs2_resblock_run_t* out, int max_runs) {
  if (!vocoder_ok(m) || stage < 0 || stage >= m->n_stages || max_runs < 0) return FS2_ERR_ARG;
  if (!stage_fused(m, stage)) return 0;
  RbRun runs[RB_MAX_RUNS];
  const int n = stage_runs(m, stage, runs);
  for (int q = 0; out && q < n && q < max_runs; q++) out[q] = runs[q];
  return n;
}

int fs2_vocoder_window_plan(const fs2_vocoder_model* m, int T, int f0, int f1, fs2_vocoder_window_launch_t* out, int max_launches) {
  if (!vocoder_ok(m) || T <= 0 || f0 < 0 || f1 <= f0 || f0 >= T || max_launches < 0 || !window_rows_ok(m, T)) return FS2_ERR_ARG;
  std::vector<fs2_vocoder_window_launch_t> L;
  FS2_TRY(window_walk(m, T, f0, f1 < T ? f1 : T, L, nullptr));
  for (int i = 0; out && i < (int)L.size() && i < max_launches; i++) out[i] = L[i];
  return (int)L.size();
}

}  // extern "C"
