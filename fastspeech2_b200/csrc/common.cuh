// Shared helpers for the fs2b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "fs2b200.h"

namespace fs2 {

extern std::atomic<unsigned long long> g_launch_count;  // host-side counter, bumped once per kernel launch (any thread)

inline int cuda_status() {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? FS2_OK : (FS2_ERR_CUDA - (int)e);
}

#define FS2_LAUNCH_CHECK()                 \
  do {                                     \
    ::fs2::g_launch_count++;               \
    int _st = ::fs2::cuda_status();        \
    if (_st != FS2_OK) return _st;         \
  } while (0)

#define FS2_TRY(expr)                      \
  do {                                     \
    int _st = (expr);                      \
    if (_st != FS2_OK) return _st;         \
  } while (0)

// Per-device one-time setup (SM count, >48 KB dynamic shared memory opt-ins).  cudaFuncSetAttribute applies to the CURRENT device's
// context, so the "done" flags are kept per device ordinal; dev_state() looks the current device up (thread-safe) and
// dev_once() runs the first-use setup per (device, kernel family).
constexpr int FS2_MAX_DEVICES = 64;
struct DevState {
  std::atomic<int> num_sms{0};
  std::atomic<bool> conv_tc_ready{false}, att_simt_ready{false}, fused_ready{false}, att_fused_ready{false}, resample_ready{false};
};
DevState* dev_state(int* err);                       // NULL + *err on failure
// Runs setup() under one process-wide lock unless `ready` is already set, and sets it when setup() succeeds.  Returns FS2_OK, or
// FS2_ERR_CUDA - e when setup() returns the error e (the next call then tries again).
int dev_once(std::atomic<bool>& ready, cudaError_t (*setup)());

// optional per-launch event timing (see fs2_profile_begin in fs2b200.h); armed per host thread
extern thread_local bool g_prof_on;
void prof_before(cudaStream_t s);
void prof_after(cudaStream_t s, int cls, double flops);

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
  switch (act) {
    case FS2_ACT_RELU: return fmaxf(v, 0.f);
    case FS2_ACT_TANH: return tanhf(v);
    case FS2_ACT_LRELU: return v > 0.f ? v : v * slope;
    default: return v;
  }
}

// Ragged batches (x_lens / lens of fs2_conv1d, fs2_resstack, fs2_conv_post): utterance b has n_b = clamp(lens[b] * scale, 0, cap) rows.
// Device lengths are clamped, never trusted.
__device__ __forceinline__ int ragged_rows(const int* lens, int scale, int cap, int b) {
  const long long n = (long long)__ldg(lens + b) * scale;
  return n <= 0 ? 0 : (n >= cap ? cap : (int)n);
}

// The rows of one vocoder layer: it computes the output rows [y0, yend) and reads input rows below xend only; rows outside the
// utterance still read as zero, so the convs pad at the utterance ends and not at the window's.  The host biases the buffer pointers
// by the windows' first rows, so kernels address window rows.  The offline layer is the window {0, cap, cap}.
struct RowWindow { int y0, yend, xend; };

// Per-utterance origin mode of the windowed layers (fs2_vocoder_forward_window and _streams): every utterance has its own window, and
// row r of the window buffers is utterance b's logical row r + org[b] * scale.  Rows stay window-relative in the kernels, so only the
// bounds move: utterance b's live rows are [lo, hi) = [-org[b] * scale, (max(lens[b], 0) - org[b]) * scale), clamped to +-ORIGIN_CAP,
// which lies beyond every window's rows (an empty span when lens[b] <= 0).  Device values are clamped, never trusted.
constexpr int ORIGIN_CAP = 1 << 30;
struct RowSpan { int lo, hi; };
__device__ __forceinline__ int origin_clamp(long long v) { return v < -ORIGIN_CAP ? -ORIGIN_CAP : (v > ORIGIN_CAP ? ORIGIN_CAP : (int)v); }
__device__ __forceinline__ RowSpan origin_rows(const int* lens, const int* org, int scale, int b) {
  const long long o = __ldg(org + b), n = max(__ldg(lens + b), 0);
  return RowSpan{origin_clamp(-o * scale), origin_clamp((n - o) * scale)};
}

// What a launcher takes in the windowed mode, NULL outside it: the layer's window rows and the utterances' origins, never one without
// the other.
struct OriginWindow { RowWindow rows; const int* org; };

// Model table: per-utterance weights, for the vocoder's multi-generator pool (fs2_vocoder_forward_streams_multi, windowed) and the
// acoustic voices mode (fs2_acoustic_{encode,decode}_voices, offline).  Row b of a launch reads its weights from model sel[b] of the
// device array of model structs (fs2_vocoder_model or fs2_acoustic_model) at `models`, `stride` bytes apart; sel is a staged table,
// always in range.  A launch names each weight it reads by a FieldRef -- the byte offset of its pointer field in the model struct and
// a float offset past that pointer -- and every row loads the pointer from its own model.  models == NULL outside these modes.
struct FieldRef { int32_t off, add; };
struct ModelTable { const unsigned char* models; const int* sel; int stride; };
// model k's weight r.  The byte offset is an int: at most FS2_MAX_GENERATORS / FS2_MAX_VOICES models of a few KB each.
__device__ __forceinline__ const float* model_weight(const ModelTable& t, int k, FieldRef r) {
  return reinterpret_cast<const float*>(__ldg(reinterpret_cast<const unsigned long long*>(t.models + (k * t.stride + r.off)))) + r.add;
}
// row b's weight r
__device__ __forceinline__ const float* row_weight(const ModelTable& t, int b, FieldRef r) { return model_weight(t, __ldg(t.sel + b), r); }
// The weights of one launch in the table mode, NULL outside it: a conv's fp32 weights, tiles and bias; a fused ResBlock launch's pairs,
// its arguments' (j, d) being ResBlock rb + j at dilation d0 + d of every generator.
struct LaunchWeights { ModelTable t; FieldRef w, wt, bias; int rb, d0; };

// A row kernel of the voices mode names up to four tables.  in (the phase's first launch only): the caller's voice indices.  That
// launch reads them itself, clamped to voice 0 outside [0, n), and stages the table the later launches read (t.sel): out[b] = the
// clamped index, out[B + b] = 1 if in[b] was in range, else 0.
struct VoiceRow { ModelTable t; FieldRef r[4]; const int* in; int n; int* out; };
__device__ __forceinline__ int voice_of(const VoiceRow& v, int b) {
  if (!v.in) return __ldg(v.t.sel + b);
  const int k = __ldg(v.in + b);
  return k >= 0 && k < v.n ? k : 0;
}
__device__ __forceinline__ const float* voice_table(const VoiceRow& v, int b, int i) { return model_weight(v.t, voice_of(v, b), v.r[i]); }
__device__ __forceinline__ void voice_stage(const VoiceRow& v, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (v.in && i < B) {
    const int k = __ldg(v.in + i);
    v.out[i] = voice_of(v, i);
    v.out[B + i] = k >= 0 && k < v.n;
  }
}

// The mel of the windowed vocoder's streams, staged by stage_mel: stream b's rows at table[b], n_mel floats apart (table != NULL), or at
// mel + b * bs, rs floats apart; its first frame f0s[b], or f0 for every stream (f0s NULL); its length lens[b] clamped to [0, cap], or
// cap (lens NULL).  ring (with table, may be NULL): stream b's frame t lives at row t mod ring[b] of table[b], and ring[b] <= 0 makes its
// length 0.
struct MelSource {
  const float* const* table;
  const float* mel; int64_t bs, rs;
  const int32_t* f0s; int f0;
  const int32_t* lens; int cap;
  const int32_t* ring;
};

// A per-element control of fs2_control_args on the [B][L] rows of a variance head or of the durations: c[b, l] = v[b * sb + l * sl]
// (strides in elements, 0 along a broadcast dimension).  rag: NULL, or the ragged mode's lengths -- columns l >= rag[b] are not read.
struct ControlView {
  const float* v; int64_t sb, sl;
  const int32_t* rag;
};

// fp32 sample -> int16 PCM as numpy's (x * scale).astype("int16") on in-range values: truncation toward zero.  Values past the int16
// range are clamped, not wrapped (fs2_wav_to_int16, fs2_resample*).
__device__ __forceinline__ short pcm16_sample(float v, float scale) {
  return (short)min(max(__float2int_rz(v * scale), -32768), 32767);
}

// ITU-T G.711 codes of an int16 PCM sample (fs2_resample_streams_mixed), as audioop.lin2ulaw / lin2alaw compute them on 16-bit input.
// mu-law: the 14-bit magnitude of s >> 2 (arithmetic), clipped to 8159 and biased by 33, lies in [32, 8192]; its segment is the position
// of its leading bit less 5 (8192, past segment 7, is the largest code), the mantissa the next four bits; every bit is inverted, the
// sign bit set for s >= 0.
__device__ __forceinline__ unsigned char ulaw_byte(short s) {
  const int v = s >> 2;
  const int mag = min(v < 0 ? -v : v, 8159) + 33;
  const int seg = 26 - __clz(mag);
  const int u = seg > 7 ? 0x7F : (seg << 4) | ((mag >> (seg + 1)) & 0xF);
  return (unsigned char)(u ^ (v < 0 ? 0x7F : 0xFF));
}

// A-law: the 13-bit s >> 3 (arithmetic), magnitude -v - 1 when negative, in [0, 4095]; segment = position of its leading bit less 4,
// at least 0; mantissa = four bits below it (bits 1..4 in segments 0 and 1); even bits inverted (xor 0x55), sign bit set for v >= 0.
__device__ __forceinline__ unsigned char alaw_byte(short s) {
  const int v = s >> 3;
  const int mag = v < 0 ? -v - 1 : v;
  const int seg = max(27 - __clz(mag), 0);
  const int a = (seg << 4) | ((mag >> (seg < 2 ? 1 : seg)) & 0xF);
  return (unsigned char)(a ^ (v < 0 ? 0x55 : 0xD5));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace fs2
