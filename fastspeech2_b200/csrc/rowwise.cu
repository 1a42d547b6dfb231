// HBM-bound row kernels: embedding + positions, speaker add, LayerNorm + pad mask, variance head
// (row dot + bucketize + embedding add), duration rounding + prefix sum, length-regulator gather,
// conv_post + tanh, and the [B,C,T] -> [B,T,C] transpose.  All fp32, float4 I/O, one warp per row.
#include "common.cuh"

namespace fs2 {

// VOICE (the row kernels' template parameter): the voices mode, vr naming the tables each utterance reads from its voice (VoiceRow).
// An instantiation of its own, so that the offline one keeps its code.

// ------------------------------------------------------------------ embedding + position (Models.py:89-91)
// Voices mode: the first launch of phase 1, which stages the voice table; r[0] the word embedding, r[1] the positions.
template <bool VOICE>
__global__ void embed_kernel(const long long* __restrict__ ids, const float* __restrict__ table,
                             const float* __restrict__ pos, float* __restrict__ y, int B, int L, int D4, int n_vocab, const VoiceRow vr) {
  if constexpr (VOICE) voice_stage(vr, B);
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * L) return;
  const int lane = threadIdx.x & 31;
  const int l = row % L;
  if constexpr (VOICE) {
    table = voice_table(vr, row / L, 0);
    pos = voice_table(vr, row / L, 1);
  }
  long long id = ids[row];
  if (id < 0 || id >= n_vocab) id = 0;  // the reference would raise; stay in bounds
  const float4* e = reinterpret_cast<const float4*>(table) + id * D4;
  const float4* p = reinterpret_cast<const float4*>(pos) + (long long)l * D4;
  float4* o = reinterpret_cast<float4*>(y) + (long long)row * D4;
  for (int c = lane; c < D4; c += 32) {
    const float4 a = __ldg(e + c), q = __ldg(p + c);
    o[c] = make_float4(a.x + q.x, a.y + q.y, a.z + q.z, a.w + q.w);
  }
}

int embed_positions(const fs2_embed_args* a, cudaStream_t s, const VoiceRow* vr) {
  if (!a || !a->ids || !a->table || !a->pos || !a->y || a->B <= 0 || a->L <= 0 || a->D <= 0) return FS2_ERR_ARG;
  if (a->D % 4) return FS2_ERR_UNSUPPORTED;
  const int rows = a->B * a->L;
  const long long* ids = reinterpret_cast<const long long*>(a->ids);
  if (vr) embed_kernel<true><<<(rows + 7) / 8, 256, 0, s>>>(ids, a->table, a->pos, a->y, a->B, a->L, a->D / 4, a->n_vocab, *vr);
  else embed_kernel<false><<<(rows + 7) / 8, 256, 0, s>>>(ids, a->table, a->pos, a->y, a->B, a->L, a->D / 4, a->n_vocab, VoiceRow{});
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ speaker add (fastspeech2.py:68-71)
// Voices mode: r[0] the speaker table
template <bool VOICE>
__global__ void rowbias_kernel(float* __restrict__ x, const float* __restrict__ table, const long long* __restrict__ idx, int B,
                               int L, int D4, int n_rows, const VoiceRow vr) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= B * L) return;
  const int lane = threadIdx.x & 31;
  if constexpr (VOICE) table = voice_table(vr, row / L, 0);
  long long id = idx[row / L];
  if (id < 0 || id >= n_rows) id = 0;
  const float4* e = reinterpret_cast<const float4*>(table) + id * D4;
  float4* o = reinterpret_cast<float4*>(x) + (long long)row * D4;
  for (int c = lane; c < D4; c += 32) {
    const float4 a = __ldg(e + c);
    float4 v = o[c];
    v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    o[c] = v;
  }
}

int add_speaker(const fs2_rowbias_args* a, cudaStream_t s, const VoiceRow* vr) {
  if (!a || !a->x || !a->table || !a->idx || a->B <= 0 || a->L <= 0 || a->D <= 0) return FS2_ERR_ARG;
  if (a->D % 4) return FS2_ERR_UNSUPPORTED;
  const int rows = a->B * a->L;
  const long long* idx = reinterpret_cast<const long long*>(a->idx);
  if (vr) rowbias_kernel<true><<<(rows + 7) / 8, 256, 0, s>>>(a->x, a->table, idx, a->B, a->L, a->D / 4, a->n_rows, *vr);
  else rowbias_kernel<false><<<(rows + 7) / 8, 256, 0, s>>>(a->x, a->table, idx, a->B, a->L, a->D / 4, a->n_rows, VoiceRow{});
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ x[b,t,:] += pos[t,:]
// Voices mode: r[0] the positions
template <bool VOICE>
__global__ void add_positions_kernel(float* __restrict__ x, const float* __restrict__ pos, long long rows, int T, int D4, const VoiceRow vr) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int t = (int)(row % T);
  if constexpr (VOICE) pos = voice_table(vr, (int)(row / T), 0);
  float4* o = reinterpret_cast<float4*>(x) + row * D4;
  const float4* p = reinterpret_cast<const float4*>(pos) + (long long)t * D4;
  for (int c = lane; c < D4; c += 32) {
    const float4 a = __ldg(p + c);
    float4 v = o[c];
    v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
    o[c] = v;
  }
}

int add_positions(float* x, const float* pos, int B, int T, int D, cudaStream_t s, const VoiceRow* vr) {
  if (!x || !pos || B <= 0 || T <= 0 || D <= 0) return FS2_ERR_ARG;
  if (D % 4) return FS2_ERR_UNSUPPORTED;
  const long long rows = (long long)B * T;
  if (vr) add_positions_kernel<true><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(x, pos, rows, T, D / 4, *vr);
  else add_positions_kernel<false><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(x, pos, rows, T, D / 4, VoiceRow{});
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ LayerNorm + pad-row zeroing
// One warp per row; the row lives in registers (C <= 1024), two-pass mean / variance like ATen's CPU kernel.
// Voices mode: r[0] gamma, r[1] beta.
template <bool VOICE>
__global__ void layernorm_kernel(const float* __restrict__ x, float* __restrict__ y, int rows, int T, int C4,
                                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                 const int* __restrict__ row_lens, int pre_relu, const VoiceRow vr) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float4* o = reinterpret_cast<float4*>(y) + (long long)row * C4;
  if (row_lens) {
    const int b = row / T, t = row - b * T;
    if (t >= row_lens[b]) {
      for (int c = lane; c < C4; c += 32) o[c] = make_float4(0.f, 0.f, 0.f, 0.f);
      return;
    }
  }
  const float4* in = reinterpret_cast<const float4*>(x) + (long long)row * C4;
  float4 v[8];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int c = lane + i * 32;
    if (c < C4) {
      v[i] = in[c];
      if (pre_relu) v[i] = make_float4(fmaxf(v[i].x, 0.f), fmaxf(v[i].y, 0.f), fmaxf(v[i].z, 0.f), fmaxf(v[i].w, 0.f));
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float inv_c = 1.f / (float)(C4 * 4);
  const float mean = warp_sum(sum) * inv_c;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int c = lane + i * 32;
    if (c < C4) {
      const float a = v[i].x - mean, b2 = v[i].y - mean, c2 = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b2 * b2) + (c2 * c2 + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) * inv_c + eps);
  if constexpr (VOICE) {
    gamma = voice_table(vr, row / T, 0);
    beta = voice_table(vr, row / T, 1);
  }
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int c = lane + i * 32;
    if (c < C4) {
      const float4 g = __ldg(g4 + c), bb = __ldg(b4 + c);
      o[c] = make_float4((v[i].x - mean) * rstd * g.x + bb.x, (v[i].y - mean) * rstd * g.y + bb.y,
                         (v[i].z - mean) * rstd * g.z + bb.z, (v[i].w - mean) * rstd * g.w + bb.w);
    }
  }
}

int layernorm(const fs2_layernorm_args* a, cudaStream_t s, const VoiceRow* vr) {
  if (!a || !a->x || !a->y || !a->gamma || !a->beta || a->B <= 0 || a->T <= 0 || a->C <= 0) return FS2_ERR_ARG;
  if (a->C % 4 || a->C > 1024) return FS2_ERR_UNSUPPORTED;
  const long long rows = (long long)a->B * a->T;
  if (rows > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
  prof_before(s);
  if (vr)
    layernorm_kernel<true><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(a->x, a->y, (int)rows, a->T, a->C / 4, a->gamma, a->beta, a->eps,
                                                                     a->row_lens, a->pre_relu, *vr);
  else
    layernorm_kernel<false><<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(a->x, a->y, (int)rows, a->T, a->C / 4, a->gamma, a->beta, a->eps,
                                                                      a->row_lens, a->pre_relu, VoiceRow{});
  prof_after(s, 2, 0.0);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ variance head (modules.py:80-100, :246-250)
// CTL: the prediction is scaled by the per-element control ctl instead of the scalar a.control (a template parameter so that the
// scalar path keeps its code and registers).  Both are one fp32 multiply: a control array of fp32(c) gives the scalar c's bits.
// Voices mode: r[0] w, r[1] b, r[2] bins, r[3] emb.
template <bool CTL, bool VOICE>
__global__ void variance_head_kernel(fs2_variance_head_args a, const ControlView ctl, const VoiceRow vr) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= a.B * a.L) return;
  const int lane = threadIdx.x & 31;
  const int b = row / a.L, l = row - b * a.L;
  if constexpr (VOICE) {
    a.w = voice_table(vr, b, 0);
    a.b = voice_table(vr, b, 1);
    if (a.bins) { a.bins = voice_table(vr, b, 2); a.emb = voice_table(vr, b, 3); }
  }
  const float4* h = reinterpret_cast<const float4*>(a.h) + (long long)row * (a.C / 4);
  const float4* w = reinterpret_cast<const float4*>(a.w);
  float acc = 0.f;
  for (int c = lane; c < a.C / 4; c += 32) {
    const float4 u = h[c], q = __ldg(w + c);
    acc += (u.x * q.x + u.y * q.y) + (u.z * q.z + u.w * q.w);
  }
  float pred = warp_sum(acc) + __ldg(a.b);
  if (a.lens && l >= a.lens[b]) pred = 0.f;  // masked_fill(mask, 0.0)
  float key = pred;
  if (a.bins) {
    if (a.target) {
      key = a.target[row];
    } else {
      if (!CTL) pred = pred * a.control;
      else if (!(ctl.rag && l >= ctl.rag[b])) pred = pred * __ldg(ctl.v + b * ctl.sb + l * ctl.sl);
      key = pred;
    }
  }
  if (lane == 0) a.pred_out[row] = pred;
  if (!a.bins) return;
  // torch.bucketize(right=False) in ATen's form: the number of edges strictly below an ordered key, and n_edges for a NaN key (no
  // edge compares >= NaN), which is the bucket the reference picks for a NaN prediction, control or target
  int lo = 0, hi = a.n_edges;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (!(__ldg(a.bins + mid) >= key)) lo = mid + 1; else hi = mid;
  }
  const float4* e = reinterpret_cast<const float4*>(a.emb) + (long long)lo * (a.D / 4);
  float4* x = reinterpret_cast<float4*>(a.x) + (long long)row * (a.D / 4);
  for (int c = lane; c < a.D / 4; c += 32) {
    const float4 q = __ldg(e + c);
    float4 v = x[c];
    v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    x[c] = v;
  }
}

// ctl: NULL or ctl->v NULL for the scalar a->control
int variance_head(const fs2_variance_head_args* a, cudaStream_t s, const ControlView* ctl, const VoiceRow* vr) {
  if (!a || !a->h || !a->w || !a->b || !a->pred_out || a->B <= 0 || a->L <= 0 || a->C <= 0) return FS2_ERR_ARG;
  if (a->C % 4) return FS2_ERR_UNSUPPORTED;
  if (a->bins && (!a->emb || !a->x || a->n_edges <= 0 || a->D <= 0 || a->D % 4)) return FS2_ERR_ARG;
  const int rows = a->B * a->L;
  const bool c = ctl && ctl->v;
  if (vr && c) variance_head_kernel<true, true><<<(rows + 7) / 8, 256, 0, s>>>(*a, *ctl, *vr);
  else if (vr) variance_head_kernel<false, true><<<(rows + 7) / 8, 256, 0, s>>>(*a, ControlView{}, *vr);
  else if (c) variance_head_kernel<true, false><<<(rows + 7) / 8, 256, 0, s>>>(*a, *ctl, VoiceRow{});
  else variance_head_kernel<false, false><<<(rows + 7) / 8, 256, 0, s>>>(*a, ControlView{}, VoiceRow{});
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ durations (modules.py:132-135, :185-187)
// One CTA per utterance: round-half-even (rintf == torch.round), truncate, block-wide inclusive scan.
// RAG: ragged batch, columns l >= src_lens[b] do not exist: they are not read, count as 0 frames and d_rounded there is 0.
// CTL: the per-element control ctl scales the rounded durations in place of the scalar a.d_control (predicted durations only).
// VOICE: voices mode: an utterance whose valid[b] is 0 (its voice index was out of range) has no columns, so 0 frames.
template <bool RAG, bool CTL, bool VOICE>
__global__ void durations_kernel(const fs2_durations_args a, const int* __restrict__ src_lens, const ControlView ctl,
                                 const int* __restrict__ valid) {
  __shared__ int warp_tot[32];
  __shared__ int carry_s;
  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int nw = blockDim.x >> 5;
  int n = RAG ? ragged_rows(src_lens, 1, a.L, b) : a.L;
  if (VOICE && !__ldg(valid + b)) n = 0;
  if (tid == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < a.L; base += blockDim.x) {
    const int l = base + tid;
    int reps = 0;
    if ((RAG || VOICE) && l >= n && l < a.L) {
      if (!a.use_target && a.d_rounded) a.d_rounded[(long long)b * a.L + l] = 0.f;
    } else if (l < a.L) {
      const float s = a.src[(long long)b * a.L + l];
      float d;
      if (a.use_target) {
        d = s;
      } else {
        const float dc = CTL ? __ldg(ctl.v + b * ctl.sb + l * ctl.sl) : a.d_control;
        const float v = rintf(expf(s) - 1.f) * dc;
        d = v <= 0.f ? 0.f : v;  // torch.clamp(min=0) keeps NaN (fmaxf would make it 0); -0 and below give +0 as fmaxf did
        if (a.d_rounded) a.d_rounded[(long long)b * a.L + l] = d;
      }
      // int() truncation toward zero.  A NaN / +-inf / absurd duration (the reference raises on int(nan) and int(+-inf), or dies
      // allocating) is counted in len_stats[2] and contributes no frames, so the caller can fail loudly instead of sizing a gigantic
      // output.
      const bool wild = !(d <= 1.0e6f && d > -INFINITY);
      if (wild) atomicAdd(a.len_stats + 2, 1);
      reps = wild ? 0 : max((int)d, 0);
    }
    int v = reps;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, v, o);
      if (lane >= o) v += n;
    }
    if (lane == 31) warp_tot[wid] = v;
    __syncthreads();
    if (wid == 0) {
      int t = lane < nw ? warp_tot[lane] : 0;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += n;
      }
      warp_tot[lane] = t;  // inclusive totals
    }
    __syncthreads();
    const int carry = carry_s;
    const int prefix = carry + (wid ? warp_tot[wid - 1] : 0) + v;
    if (l < a.L) a.cum[(long long)b * a.L + l] = prefix;
    __syncthreads();
    if (tid == 0) carry_s = carry + warp_tot[nw - 1];
    __syncthreads();
  }
  if (tid == 0) {
    const int total = carry_s;
    a.mel_lens[b] = total;
    if (a.mel_lens32) a.mel_lens32[b] = total;
    atomicMax(a.len_stats, total);
    atomicAdd(a.len_stats + 1, total);
  }
}

// src_lens: the ragged mode's lengths or NULL.  ctl: NULL or ctl->v NULL for the scalar a->d_control; ignored with use_target.
// valid: NULL, or the voices mode's validity flags.
int durations(const fs2_durations_args* a, cudaStream_t s, const int32_t* src_lens, const ControlView* ctl, const int32_t* valid) {
  if (!a || !a->src || !a->cum || !a->mel_lens || !a->len_stats || a->B <= 0 || a->L <= 0) return FS2_ERR_ARG;
  cudaError_t e = cudaMemsetAsync(a->len_stats, 0, 3 * sizeof(int), s);
  if (e != cudaSuccess) return FS2_ERR_CUDA - (int)e;
  const ControlView c = (ctl && !a->use_target) ? *ctl : ControlView{};
  if (valid) {
    if (c.v) {
      if (src_lens) durations_kernel<true, true, true><<<a->B, 256, 0, s>>>(*a, src_lens, c, valid);
      else durations_kernel<false, true, true><<<a->B, 256, 0, s>>>(*a, nullptr, c, valid);
    } else {
      if (src_lens) durations_kernel<true, false, true><<<a->B, 256, 0, s>>>(*a, src_lens, c, valid);
      else durations_kernel<false, false, true><<<a->B, 256, 0, s>>>(*a, nullptr, c, valid);
    }
  } else if (c.v) {
    if (src_lens) durations_kernel<true, true, false><<<a->B, 256, 0, s>>>(*a, src_lens, c, nullptr);
    else durations_kernel<false, true, false><<<a->B, 256, 0, s>>>(*a, nullptr, c, nullptr);
  } else {
    if (src_lens) durations_kernel<true, false, false><<<a->B, 256, 0, s>>>(*a, src_lens, c, nullptr);
    else durations_kernel<false, false, false><<<a->B, 256, 0, s>>>(*a, nullptr, c, nullptr);
  }
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ y0[b,t,:] = y1[b,t,:] = 0 for t >= lens[b] (ragged acoustic outputs)
__global__ void zero_tail_kernel(float* __restrict__ y0, float* __restrict__ y1, const int* __restrict__ lens, long long rows, int T, int C4) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int b = (int)(row / T), t = (int)(row - (long long)b * T);
  if (t < ragged_rows(lens, 1, T, b)) return;
  const int lane = threadIdx.x & 31;
  float4* o0 = reinterpret_cast<float4*>(y0) + row * C4;
  float4* o1 = reinterpret_cast<float4*>(y1) + row * C4;
  for (int c = lane; c < C4; c += 32) { o0[c] = make_float4(0.f, 0.f, 0.f, 0.f); o1[c] = make_float4(0.f, 0.f, 0.f, 0.f); }
}

int zero_tail(float* y0, float* y1, const int32_t* lens, int B, int T, int C, cudaStream_t s) {
  if (!y0 || !y1 || !lens || B <= 0 || T <= 0 || C <= 0) return FS2_ERR_ARG;
  if (C % 4 || !aligned16(y0) || !aligned16(y1)) return FS2_ERR_UNSUPPORTED;
  const long long rows = (long long)B * T;
  zero_tail_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(y0, y1, lens, rows, T, C / 4);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ length regulator gather (modules.py:167-194)
// One warp per output frame: binary search of the inclusive duration prefix sums (L2/L1 resident, 4*L bytes per utterance),
// then a coalesced float4 copy of the source phoneme row with the decoder position row added (Models.py:158-160).
// Voices mode: the first launch of phase 2, which stages the voice table; r[0] the positions.
template <bool VOICE>
__global__ void length_regulate_kernel(fs2_length_regulate_args a, const VoiceRow vr) {
  if constexpr (VOICE) voice_stage(vr, a.B);
  const long long frame = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (frame >= (long long)a.B * a.T) return;
  const int lane = threadIdx.x & 31;
  const int b = (int)(frame / a.T), t = (int)(frame - (long long)b * a.T);
  if constexpr (VOICE) if (a.pos) a.pos = voice_table(vr, b, 0);
  const int* cum = a.cum + (long long)b * a.L;
  const int total = __ldg(cum + a.L - 1);
  const int D4 = a.D / 4;
  float4* o = reinterpret_cast<float4*>(a.y) + frame * D4;
  const float4* pos = a.pos ? reinterpret_cast<const float4*>(a.pos) + (long long)t * D4 : nullptr;
  if (t >= total) {
    for (int c = lane; c < D4; c += 32) o[c] = pos ? __ldg(pos + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  int lo = 0, hi = a.L - 1;  // first i with cum[i] > t
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(cum + mid) > t) hi = mid; else lo = mid + 1;
  }
  const float4* src = reinterpret_cast<const float4*>(a.x) + ((long long)b * a.L + lo) * D4;
  for (int c = lane; c < D4; c += 32) {
    float4 v = __ldg(src + c);
    if (pos) {
      const float4 q = __ldg(pos + c);
      v.x += q.x; v.y += q.y; v.z += q.z; v.w += q.w;
    }
    o[c] = v;
  }
}

int length_regulate(const fs2_length_regulate_args* a, cudaStream_t s, const VoiceRow* vr) {
  if (!a || !a->x || !a->cum || !a->y || a->B <= 0 || a->L <= 0 || a->T <= 0 || a->D <= 0) return FS2_ERR_ARG;
  if (a->D % 4) return FS2_ERR_UNSUPPORTED;
  const long long frames = (long long)a->B * a->T;
  prof_before(s);
  if (vr) length_regulate_kernel<true><<<(unsigned)((frames + 7) / 8), 256, 0, s>>>(*a, *vr);
  else length_regulate_kernel<false><<<(unsigned)((frames + 7) / 8), 256, 0, s>>>(*a, VoiceRow{});
  prof_after(s, 3, 0.0);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ conv_post + tanh (hifigan/models.py:161-163)
// C_in = 32, one output channel: 128 B per input row, HBM-bound (algorithmic traffic = one read of x).  A CTA stages
// 256 + taps - 1 activated rows in shared memory with fully coalesced float4 loads (row stride C+1 floats -> conflict-free
// column walks), then each thread reduces its own output sample from shared memory.
constexpr int CP_ROWS = 256;
// Batch strides of x and wav and the rows computed and read: {T * C, T} and {0, T, T} outside the windowed mode (RowWindow; x / wav
// are then biased by the windows' first rows).
// org: NULL, or the windowed mode's per-utterance origins (origin_rows): rows and samples outside [lo_b, hi_b) read and write zero.
// lw: the table mode's weights (the *_streams_multi_kernel entry points): w and bias of utterance b's generator.
struct PostRows { long long xbs, wbs; RowWindow win; const int* org; LaunchWeights lw; };
// The conv's weights and bias: the call's, or in the table mode those of utterance b's generator
template <bool MULTI>
__device__ __forceinline__ void conv_post_weights(const fs2_conv_post_args& a, const PostRows& pr, int b, const float*& w, const float*& bias) {
  w = a.w; bias = a.bias;
  if constexpr (MULTI) {
    w = row_weight(pr.lw.t, b, pr.lw.w);
    bias = row_weight(pr.lw.t, b, pr.lw.bias);
  }
}
template <bool ORG, bool MULTI = false>
__device__ __forceinline__ void conv_post_body(const fs2_conv_post_args a, int tiles_per_batch, const PostRows pr) {
  extern __shared__ float cp_smem[];
  const int C = a.C, ld = C + 1, pad = (a.taps - 1) / 2;
  float* wsm = cp_smem;                   // [taps][C]
  float* xs = cp_smem + a.taps * C;       // [CP_ROWS + taps - 1][C + 1]
  const int b = blockIdx.x / tiles_per_batch;
  const int t0 = pr.win.y0 + (blockIdx.x % tiles_per_batch) * CP_ROWS;
  int n_b, lo_b = 0;
  if constexpr (ORG) {
    const RowSpan r = origin_rows(a.lens, pr.org, a.lens_scale, b);
    n_b = r.hi; lo_b = r.lo;
  } else {
    n_b = a.lens ? ragged_rows(a.lens, a.lens_scale, a.T, b) : a.T;   // ragged batch: rows >= n_b read as zero, wav there is 0
  }
  const int nin = min(n_b, pr.win.xend);
  const float *w, *bias;
  conv_post_weights<MULTI>(a, pr, b, w, bias);
  for (int i = threadIdx.x; i < a.taps * C; i += blockDim.x) wsm[i] = w[i];
  const int rows = CP_ROWS + a.taps - 1, C4 = C / 4;
  const float* xf = a.x + (long long)b * pr.xbs;
  const float4* xb = reinterpret_cast<const float4*>(xf);
  // x need not be 16-byte aligned here (the dispatcher sends such an x to this kernel, e.g. a view at an odd float offset): scalar loads
  const bool vec = (reinterpret_cast<uintptr_t>(xf) & 15u) == 0;
  for (int i = threadIdx.x; i < rows * C4; i += blockDim.x) {
    const int r = i / C4, c4 = i - r * C4;
    const int t = t0 - pad + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    bool in;
    if constexpr (ORG) in = t >= lo_b && t < nin;
    else in = t >= 0 && t < nin;
    if (in) {
      if (vec) {
        v = __ldg(xb + (long long)t * C4 + c4);
      } else {
        const float* p = xf + (long long)t * C + c4 * 4;
        v = make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), __ldg(p + 3));
      }
      v.x = v.x > 0.f ? v.x : v.x * a.in_slope;
      v.y = v.y > 0.f ? v.y : v.y * a.in_slope;
      v.z = v.z > 0.f ? v.z : v.z * a.in_slope;
      v.w = v.w > 0.f ? v.w : v.w * a.in_slope;
    }
    float* d = xs + r * ld + c4 * 4;
    d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
  }
  __syncthreads();
  const int t = t0 + threadIdx.x;
  if (t >= pr.win.yend) return;
  float acc = __ldg(bias);
  for (int j = 0; j < a.taps; j++) {
    const float* xr = xs + (threadIdx.x + j) * ld;
    const float* wj = wsm + j * C;
#pragma unroll 8
    for (int c = 0; c < C; c++) acc = fmaf(xr[c], wj[c], acc);
  }
  a.wav[(long long)b * pr.wbs + t] = (t < n_b && (!ORG || t >= lo_b)) ? tanhf(acc) : 0.f;
}

__global__ void __launch_bounds__(CP_ROWS) conv_post_kernel(const fs2_conv_post_args a, int tiles_per_batch, const PostRows pr) {
  conv_post_body<false>(a, tiles_per_batch, pr);
}
// Windowed mode (fs2_vocoder_forward_window and _streams): entry points of their own, so that the offline ones keep their code
__global__ void __launch_bounds__(CP_ROWS) conv_post_streams_kernel(const fs2_conv_post_args a, int tiles_per_batch, const PostRows pr) {
  conv_post_body<true>(a, tiles_per_batch, pr);
}
__global__ void __launch_bounds__(CP_ROWS) conv_post_streams_multi_kernel(const fs2_conv_post_args a, int tiles_per_batch, const PostRows pr) {
  conv_post_body<true, true>(a, tiles_per_batch, pr);
}

// The generator's own shape (32 channels, 7 taps, hifigan/models.py:131): no shared memory at all.  Eight lanes own one time row (one
// float4 of channels each: a warp reads 4 full 128-byte lines per load instruction, each row exactly once per group plus a 6-row halo),
// the 7 x 4 weights of a lane live in registers, and TAPS sliding accumulators carry the partial sums of the outputs a row contributes to;
// a finished output is reduced over the 8 lanes by three shuffles and every lane keeps one of 8 consecutive samples, so the stores are
// full 32-byte sectors.  (The staged kernel above issues two shared-memory loads per FMA and measured 263 us = 2.0 TB/s at
// B = 16 x 259k samples; this one is bound by the single read of x.)
constexpr int CPF_BLOCKS = 18;                         // row blocks of TAPS rows per 8-lane group
// RAG: ragged batch (a.lens != NULL); a template parameter so that the padded path keeps its code and registers.  ORG (with RAG): the
// windowed mode's per-utterance origins.  MULTI (with ORG): the multi-generator mode.
template <int TAPS, bool RAG, bool ORG, bool MULTI = false>
__device__ __forceinline__ void conv_post_c32_body(const fs2_conv_post_args a, int groups_per_batch, long long n_groups, const PostRows pr) {
  constexpr int PAD = (TAPS - 1) / 2, ROWS = CPF_BLOCKS * TAPS - 2 * PAD;     // output rows per group (120 for 7 taps: a multiple of 8)
  static_assert(ROWS % 8 == 0, "full 8-sample stores");
  const int lane = threadIdx.x & 31, sub = lane & 7;
  long long grp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const bool live = grp < n_groups;                     // groups past the end run along with an empty row range (full-warp shuffles below)
  grp = live ? grp : 0;
  const int b = (int)(grp / groups_per_batch);
  const int t0 = pr.win.y0 + (int)(grp - (long long)b * groups_per_batch) * ROWS;
  const int T = live ? a.T : 0;
  const int tend = min(t0 + ROWS, live ? pr.win.yend : 0);
  int n_b, lo_b = 0;
  if constexpr (ORG) {
    const RowSpan r = origin_rows(a.lens, pr.org, a.lens_scale, b);
    n_b = live ? r.hi : 0; lo_b = live ? r.lo : 0;
  } else {
    n_b = RAG ? ragged_rows(a.lens, a.lens_scale, T, b) : T;   // ragged batch: rows >= n_b read as zero, wav there is 0
  }
  const int nin = min(n_b, pr.win.xend);
  const float *wp, *bp;
  conv_post_weights<MULTI>(a, pr, b, wp, bp);
  float4 w[TAPS];
#pragma unroll
  for (int j = 0; j < TAPS; j++) w[j] = __ldg(reinterpret_cast<const float4*>(wp + j * 32) + sub);
  const float bias = __ldg(bp), slope = a.in_slope;
  const float4* xb = reinterpret_cast<const float4*>(a.x + (long long)b * pr.xbs) + sub;
  float* wb = a.wav + (long long)b * pr.wbs;
  float s[TAPS];
#pragma unroll
  for (int k = 0; k < TAPS; k++) s[k] = 0.f;
  float keep = 0.f;
#pragma unroll 1
  for (int blk = 0; blk < CPF_BLOCKS; blk++) {
    const int rb = t0 - PAD + blk * TAPS;
    float4 x[TAPS];
#pragma unroll
    for (int i = 0; i < TAPS; i++) {
      const int r = rb + i;
      x[i] = (r >= lo_b && r < nin) ? __ldg(xb + (long long)r * 8) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < TAPS; i++) {
      float4 v = x[i];
      v.x = v.x > 0.f ? v.x : v.x * slope; v.y = v.y > 0.f ? v.y : v.y * slope;
      v.z = v.z > 0.f ? v.z : v.z * slope; v.w = v.w > 0.f ? v.w : v.w * slope;
      // row r feeds outputs r - PAD .. r + PAD; s[k] is the partial sum of output r - PAD + k, which takes tap TAPS - 1 - k of this row
#pragma unroll
      for (int k = 0; k < TAPS; k++) {
        const float4 wj = w[TAPS - 1 - k];
        s[k] = fmaf(v.x, wj.x, fmaf(v.y, wj.y, fmaf(v.z, wj.z, fmaf(v.w, wj.w, s[k]))));
      }
      float tot = s[0];                                 // output r - PAD has received its last row
#pragma unroll
      for (int k = 0; k + 1 < TAPS; k++) s[k] = s[k + 1];
      s[TAPS - 1] = 0.f;
      tot += __shfl_xor_sync(0xffffffffu, tot, 4);
      tot += __shfl_xor_sync(0xffffffffu, tot, 2);
      tot += __shfl_xor_sync(0xffffffffu, tot, 1);
      const int t = rb + i - PAD;
      if (t >= t0 && t < tend) {
        const int o = (t - t0) & 7;
        if (o == sub) keep = tot;
        if (o == 7 || t == tend - 1) {
          if (sub <= o) wb[t - o + sub] = (!RAG || (t - o + sub < n_b && (!ORG || t - o + sub >= lo_b))) ? tanhf(keep + bias) : 0.f;
        }
      }
    }
  }
}

template <int TAPS, bool RAG>
__global__ void __launch_bounds__(256) conv_post_c32_kernel(const fs2_conv_post_args a, int groups_per_batch, long long n_groups, const PostRows pr) {
  conv_post_c32_body<TAPS, RAG, false>(a, groups_per_batch, n_groups, pr);
}
template <int TAPS>
__global__ void __launch_bounds__(256) conv_post_c32_streams_kernel(const fs2_conv_post_args a, int groups_per_batch, long long n_groups,
                                                                    const PostRows pr) {
  conv_post_c32_body<TAPS, true, true>(a, groups_per_batch, n_groups, pr);
}
template <int TAPS>
__global__ void __launch_bounds__(256) conv_post_c32_streams_multi_kernel(const fs2_conv_post_args a, int groups_per_batch, long long n_groups,
                                                                          const PostRows pr) {
  conv_post_c32_body<TAPS, true, true, true>(a, groups_per_batch, n_groups, pr);
}

// win (with a->lens): NULL, or the windowed mode (OriginWindow; a->T is not used, a->x and a->wav are biased by the windows' first rows
// and their batch strides are x_bs and wav_bs).  Both kernels add every output's taps in the same order wherever its tile starts.
// lw (with win): NULL, or the table mode (LaunchWeights): a->w and a->bias are model 0's.
int conv_post(const fs2_conv_post_args* a, cudaStream_t s, const OriginWindow* win, const LaunchWeights* lw, long long x_bs, long long wav_bs) {
  if (!a || !a->x || !a->w || !a->bias || !a->wav || a->B <= 0 || a->T <= 0 || a->C <= 0 || a->taps <= 0) return FS2_ERR_ARG;
  if (a->lens && a->lens_scale < 1) return FS2_ERR_ARG;
  if (win && !a->lens) return FS2_ERR_ARG;
  if (lw && !win) return FS2_ERR_UNSUPPORTED;           // the table mode's entry points are windowed
  const PostRows pr = win ? PostRows{x_bs, wav_bs, win->rows, win->org, lw ? *lw : LaunchWeights{}}
                          : PostRows{(long long)a->T * a->C, a->T, RowWindow{0, a->T, a->T}, nullptr, LaunchWeights{}};
  const int rows = pr.win.yend - pr.win.y0;
  if (rows <= 0) return FS2_ERR_ARG;
  if (a->C == 32 && a->taps == 7 && (reinterpret_cast<uintptr_t>(a->x) & 15u) == 0 && (reinterpret_cast<uintptr_t>(a->w) & 15u) == 0) {
    constexpr int ROWS = CPF_BLOCKS * 7 - 6;
    const int gpb = (rows + ROWS - 1) / ROWS;
    const long long n_groups = (long long)gpb * a->B, blocks = (n_groups * 8 + 255) / 256;
    if (blocks > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
    prof_before(s);
    if (lw) conv_post_c32_streams_multi_kernel<7><<<(unsigned)blocks, 256, 0, s>>>(*a, gpb, n_groups, pr);
    else if (win) conv_post_c32_streams_kernel<7><<<(unsigned)blocks, 256, 0, s>>>(*a, gpb, n_groups, pr);
    else if (a->lens) conv_post_c32_kernel<7, true><<<(unsigned)blocks, 256, 0, s>>>(*a, gpb, n_groups, pr);
    else conv_post_c32_kernel<7, false><<<(unsigned)blocks, 256, 0, s>>>(*a, gpb, n_groups, pr);
    prof_after(s, 3, 2.0 * (double)a->B * rows * a->taps * a->C);
    FS2_LAUNCH_CHECK();
    return FS2_OK;
  }
  const size_t smem = ((size_t)a->taps * a->C + (size_t)(CP_ROWS + a->taps - 1) * (a->C + 1)) * sizeof(float);
  if (a->C % 4 || smem > 48 * 1024) return FS2_ERR_UNSUPPORTED;
  const int tiles = (rows + CP_ROWS - 1) / CP_ROWS;
  const long long n = (long long)a->B * rows;
  if ((long long)tiles * a->B > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
  prof_before(s);
  if (lw) conv_post_streams_multi_kernel<<<(unsigned)(tiles * a->B), CP_ROWS, smem, s>>>(*a, tiles, pr);
  else if (win) conv_post_streams_kernel<<<(unsigned)(tiles * a->B), CP_ROWS, smem, s>>>(*a, tiles, pr);
  else conv_post_kernel<<<(unsigned)(tiles * a->B), CP_ROWS, smem, s>>>(*a, tiles, pr);
  prof_after(s, 3, 2.0 * n * a->taps * a->C);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ mel staging of the windowed vocoder
// out[b][r] = stream b's mel row o_b + x0 + r for r < rows, zeros where that row lies outside [0, n_b), with o_b and n_b the origin and
// length of MelSource; org[b] = o_b and lens[b] = n_b.  The one kernel that reads the caller's mel and lengths, so the window kernels
// after it see one batch-strided buffer and two tables.  n_mel % 4 == 0 and 16-byte aligned rows (float4 loads); rows outside the
// utterance are never dereferenced, and a ring's rows are read at t mod ring[b] only.  MULTI: gen[b] = stream b's generator index
// gen_in[b], or 0 -- and length 0 -- for one outside [0, n_gen), so that the window kernels index the generators with it unchecked.
template <bool MULTI>
__device__ __forceinline__ void stage_mel_body(const MelSource& src, int B, int x0, int rows, int n4, float4* out, int* org, int* lens,
                                               const int* gen_in, int n_gen, int* gen, long long total) {
  auto origin = [&](int b) { return src.f0s ? __ldg(src.f0s + b) : src.f0; };
  auto gen_ok = [&](int b) {
    if constexpr (MULTI) {
      const int g = __ldg(gen_in + b);
      return g >= 0 && g < n_gen;
    }
    return true;
  };
  auto length = [&](int b) {
    if (src.ring && __ldg(src.ring + b) <= 0) return 0;
    if (!gen_ok(b)) return 0;
    return src.lens ? min(max(__ldg(src.lens + b), 0), src.cap) : src.cap;
  };
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long br = i / n4;
    const int c4 = (int)(i - br * n4);
    const int b = (int)(br / rows), r = (int)(br - (long long)b * rows);
    const long long t = (long long)origin(b) + x0 + r;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t >= 0 && t < length(b)) {
      const long long tr = src.ring ? t % __ldg(src.ring + b) : t;     // length(b) > 0 implies ring[b] > 0
      const float* row = src.table ? src.table[b] + tr * n4 * 4 : src.mel + b * src.bs + t * src.rs;
      v = __ldg(reinterpret_cast<const float4*>(row) + c4);
    }
    out[i] = v;
    if (i < B) {
      org[i] = origin((int)i); lens[i] = length((int)i);
      if constexpr (MULTI) gen[i] = gen_ok((int)i) ? __ldg(gen_in + i) : 0;
    }
  }
}
__global__ void stage_mel_kernel(const MelSource src, int B, int x0, int rows, int n4, float4* out, int* org, int* lens, long long total) {
  stage_mel_body<false>(src, B, x0, rows, n4, out, org, lens, nullptr, 0, nullptr, total);
}
__global__ void stage_mel_multi_kernel(const MelSource src, int B, int x0, int rows, int n4, float4* out, int* org, int* lens,
                                       const int* gen_in, int n_gen, int* gen, long long total) {
  stage_mel_body<true>(src, B, x0, rows, n4, out, org, lens, gen_in, n_gen, gen, total);
}

// gen: NULL, or the multi-generator mode's staged table of gen_in's n_gen generators (src.table set)
int stage_mel(const MelSource& src, int B, int x0, int rows, int n_mel, float* out, int32_t* org, int32_t* lens, const int32_t* gen_in,
              int n_gen, int32_t* gen, cudaStream_t s) {
  if (!(src.table || src.mel) || (src.ring && !src.table) || !out || !org || !lens || B <= 0 || rows <= 0 || n_mel <= 0) return FS2_ERR_ARG;
  if (gen && !(gen_in && src.table)) return FS2_ERR_ARG;
  if (n_mel % 4 || !aligned16(out) || (!src.table && ((src.bs | src.rs) & 3))) return FS2_ERR_UNSUPPORTED;
  if (!src.table && !aligned16(src.mel)) return FS2_ERR_ARG;
  const long long total = (long long)B * rows * (n_mel / 4);
  const long long blocks = (total + 255) / 256;
  prof_before(s);
  const unsigned grid = (unsigned)(blocks < 4096 ? blocks : 4096);
  if (gen)
    stage_mel_multi_kernel<<<grid, 256, 0, s>>>(src, B, x0, rows, n_mel / 4, reinterpret_cast<float4*>(out), org, lens, gen_in, n_gen, gen, total);
  else stage_mel_kernel<<<grid, 256, 0, s>>>(src, B, x0, rows, n_mel / 4, reinterpret_cast<float4*>(out), org, lens, total);
  prof_after(s, 3, 0.0);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ appending arriving mel frames to the streams' rings
// Block (r, y) copies its share of record r's frames, one float4 (four channels of one frame) per element: channels fastest from a
// channels-last source (float4 loads and stores both coalesced), frames fastest from any other (a channel-major block's four scalar
// loads are then coalesced along its frames).  Only the last cap frames of a longer record are copied, so no two elements of a record
// store to the same ring row.
__global__ void mel_ring_append_kernel(const fs2_mel_ring_record_t* __restrict__ table, int n4, int max_count) {
  const fs2_mel_ring_record_t rec = table[blockIdx.x];
  const int cap = rec.cap;
  if (cap <= 0 || (reinterpret_cast<uintptr_t>(rec.ring) & 15u)) return;
  const int cnt = min(max(rec.count, 0), max_count);
  const int skip = cnt > cap ? cnt - cap : 0, frames = cnt - skip;
  const long long fs = rec.frame_stride, cs = rec.channel_stride;
  const bool vec = cs == 1 && (fs & 3) == 0 && (reinterpret_cast<uintptr_t>(rec.src) & 15u) == 0;
  const long long total = (long long)frames * n4;
  for (long long e = (long long)blockIdx.y * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.y * blockDim.x) {
    const int i = skip + (int)(vec ? e / n4 : e % frames), c4 = (int)(vec ? e % n4 : e / frames);
    const float* s = rec.src + (rec.src_frame + i) * fs + (long long)c4 * 4 * cs;
    float4 v;
    if (vec) {
      v = __ldg(reinterpret_cast<const float4*>(s));
    } else {
      v.x = __ldg(s); v.y = __ldg(s + cs); v.z = __ldg(s + 2 * cs); v.w = __ldg(s + 3 * cs);
    }
    long long row = (rec.dst_frame + i) % cap;
    if (row < 0) row += cap;
    reinterpret_cast<float4*>(rec.ring + row * n4 * 4)[c4] = v;
  }
}

int mel_ring_append(const fs2_mel_ring_append_args* a, cudaStream_t s) {
  if (!a || !a->table || a->n_records <= 0 || a->max_count <= 0) return FS2_ERR_ARG;
  if (a->n_mel <= 0 || a->n_mel % 4) return FS2_ERR_UNSUPPORTED;
  const int n4 = a->n_mel / 4;
  const long long per = ((long long)a->max_count * n4 + 255) / 256;
  prof_before(s);
  mel_ring_append_kernel<<<dim3((unsigned)a->n_records, (unsigned)(per < 65535 ? per : 65535)), 256, 0, s>>>(a->table, n4, a->max_count);
  prof_after(s, 3, 0.0);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ [B,C,T] -> [B,T,C]
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int T) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float* ib = in + (long long)b * C * T;
  float* ob = out + (long long)b * C * T;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    if (c < C && t < T) tile[i][threadIdx.x] = ib[(long long)c * T + t];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (c < C && t < T) ob[(long long)t * C + c] = tile[threadIdx.x][i];
  }
}

int transpose_bct_to_btc(const float* in, float* out, int B, int C, int T, cudaStream_t s) {
  if (!in || !out || B <= 0 || C <= 0 || T <= 0) return FS2_ERR_ARG;
  dim3 grid((T + 31) / 32, (C + 31) / 32, B), block(32, 8);
  transpose_kernel<<<grid, block, 0, s>>>(in, out, C, T);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

// ------------------------------------------------------------------ waveform -> int16 + per-utterance trim (utils/model.py:82-90)
// out[b][t] = t < lens[b] ? (int16) trunc(wav[b][t] * scale) : 0.  numpy's astype("int16") truncates toward zero; values beyond the
// int16 range (|wav| >= 1 after tanh: not reachable) are clamped instead of wrapping.  One thread converts 8 samples (16-byte store).
__global__ void wav_to_int16_kernel(const float* __restrict__ wav, long long wav_bs, const long long* __restrict__ lens, float scale, int B,
                                    long long N, short* __restrict__ out) {
  const long long per_b = (N + 7) / 8;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= per_b * B) return;
  const int b = (int)(idx / per_b);
  const long long t0 = (idx - (long long)b * per_b) * 8;
  const long long len = lens ? min(max(lens[b], 0LL), N) : N;
  const float* src = wav + (long long)b * wav_bs + t0;
  short v[8];
  if (t0 + 8 <= N && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0)) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(src)), c = __ldg(reinterpret_cast<const float4*>(src) + 1);
    const float f[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = t0 + k < len ? pcm16_sample(f[k], scale) : (short)0;
  } else {
#pragma unroll
    for (int k = 0; k < 8; k++) v[k] = (t0 + k < N && t0 + k < len) ? pcm16_sample(src[k], scale) : (short)0;
  }
  short* dst = out + (long long)b * N + t0;
  if (t0 + 8 <= N && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(v);
  } else {
    for (int k = 0; k < 8 && t0 + k < N; k++) dst[k] = v[k];
  }
}

int wav_to_int16(const fs2_wav_int16_args* a, cudaStream_t s) {
  if (!a || !a->wav || !a->out || a->B <= 0 || a->N <= 0) return FS2_ERR_ARG;
  const long long threads = ((a->N + 7) / 8) * a->B;
  wav_to_int16_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(a->wav, (long long)a->wav_batch_stride, reinterpret_cast<const long long*>(a->lens), a->scale, a->B, (long long)a->N, reinterpret_cast<short*>(a->out));
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
