// Polyphase FIR sample-rate conversion of the waveform: scipy.signal.resample_poly's arithmetic in fp32 (include/fs2b200.h).
// One kernel serves the offline, window, streams and mixed streams calls; they differ only in where a row's input pieces, length,
// output range, filter and encoding come from (RsRow).  The first three are the one-filter case of the mixed call's table.
#include <algorithm>
#include <cstddef>

#include "common.cuh"

namespace fs2 {

constexpr int RS_THREADS = 256, RS_R = 8, RS_J = RS_THREADS * RS_R;   // outputs per tile: RS_R per thread
constexpr int RS_CHUNK_MAX = 8192;                                     // input floats staged per pass

// One filter: [up][K] taps at row stride Kp, and the inputs staged per pass (chunk)
struct RsFilter {
  int up, down, K, Kp, half_len, chunk;
  const float* taps;
};

// One row: input samples [i0, i1) at x0, [i1, i2) at x1, n samples in all (inputs outside [0, n) are zero); outputs [j0, j0 + cnt)
// go to y[j - j0] in encoding enc, through filter `filter`.
struct RsRow {
  const float *x0, *x1;
  long long i0, i1, i2, n, j0, cnt;
  void* y;
  int filter, enc;
};

struct RsParams {
  RsFilter f[FS2_RESAMPLE_MAX_FILTERS]; int n_filters;
  int enc; float scale;                  // enc: every row's encoding in the offline, window and streams calls
  // offline and window calls: pieces shared by every row, with batch strides
  const float *x0, *x1; long long x0_bs, x1_bs, i0, i1, i2, N, j0, j1;
  const int32_t* lens; int lens_scale;
  void* y; long long y_bs;
  // streams and mixed calls: a device record per row
  const fs2_resample_stream_t* table; const fs2_resample_mixed_stream_t* mixed; long long max_out;
};

__host__ __device__ __forceinline__ int rs_elem_bytes(int enc) {
  return enc == FS2_RESAMPLE_F32 ? 4 : enc == FS2_RESAMPLE_PCM16 ? 2 : 1;
}

__device__ __forceinline__ RsRow rs_row(const RsParams& P, int b) {
  RsRow r;
  if (P.mixed) {
    const fs2_resample_mixed_stream_t* t = P.mixed + b;
    r.x0 = t->x0; r.x1 = t->x1;
    r.i0 = t->i0; r.i1 = t->i1; r.i2 = t->i2;
    r.n = max((long long)t->n, 0LL);
    r.j0 = t->j0;
    r.cnt = min(max((long long)(t->j1 - t->j0), 0LL), P.max_out);
    r.filter = t->filter; r.enc = t->encoding;
    const long long off = t->y_offset;
    r.y = static_cast<char*>(P.y) + off;
    if (r.filter < 0 || r.filter >= P.n_filters || r.enc < FS2_RESAMPLE_F32 || r.enc > FS2_RESAMPLE_ALAW || off < 0 || (off & 15)) {
      r.cnt = 0;                                                           // outside the table: write nothing
      r.filter = 0;
    }
    return r;
  }
  r.filter = 0; r.enc = P.enc;
  r.y = static_cast<char*>(P.y) + (size_t)b * P.y_bs * rs_elem_bytes(P.enc);
  if (P.table) {
    const fs2_resample_stream_t* t = P.table + b;
    r.x0 = t->x0; r.x1 = t->x1;
    r.i0 = t->i0; r.i1 = t->i1; r.i2 = t->i2;
    r.n = max((long long)t->n, 0LL);
    r.j0 = t->j0;
    r.cnt = min(max((long long)(t->j1 - t->j0), 0LL), P.max_out);
  } else {
    r.x0 = P.x0 ? P.x0 + (long long)b * P.x0_bs : nullptr;
    r.x1 = P.x1 ? P.x1 + (long long)b * P.x1_bs : nullptr;
    r.i0 = P.i0; r.i1 = P.i1; r.i2 = P.i2;
    r.n = P.lens ? min(max((long long)__ldg(P.lens + b) * P.lens_scale, 0LL), P.N) : P.N;
    r.j0 = P.j0;
    r.cnt = P.j1 - P.j0;
  }
  return r;
}

__device__ __forceinline__ float rs_input(const RsRow& r, long long i) {
  if (i < 0 || i >= r.n) return 0.f;
  if (i >= r.i0 && i < r.i1 && r.x0) return __ldg(r.x0 + (i - r.i0));
  if (i >= r.i1 && i < r.i2 && r.x1) return __ldg(r.x1 + (i - r.i1));
  return 0.f;   // not provided: the host proves such inputs unneeded (window call) or leaves them to the caller (streams call)
}

// grid (tiles, rows).  Each block copies its row's [up][K] taps to shared memory once (row stride Kp = K | 1, odd, so that the phases
// of a warp's 32 consecutive outputs spread over the banks) and then walks its row's tiles of RS_J outputs.  Per tile it stages the
// input span of the tile's outputs in shared memory, in passes of at most `chunk` samples, so that adjacent outputs share their input
// loads from global memory; thread t owns outputs t + 256 r (r < RS_R), so loads, stores and tap reads of a warp are consecutive.
// Each output accumulates its taps in ascending input order across the passes.  The filter is the row's, read from the parameter
// table: unbounded, its fields in registers would take the kernel from 80 to 114 registers and 3 to 2 blocks per SM, so the bound
// keeps 3 (77 registers, no spills).
__global__ void __launch_bounds__(RS_THREADS, 3) resample_kernel(const RsParams P) {
  extern __shared__ float smem[];
  const RsRow r = rs_row(P, blockIdx.y);
  const long long n_tiles = (r.cnt + RS_J - 1) / RS_J;
  if ((long long)blockIdx.x >= n_tiles) return;
  const RsFilter& F = P.f[r.filter];
  const int up = F.up, down = F.down, K = F.K, Kp = F.Kp, half_len = F.half_len, chunk = F.chunk;
  float* taps = smem;
  float* xs = smem + up * Kp;
  for (int e = threadIdx.x; e < up * K; e += RS_THREADS) taps[(e / K) * Kp + e % K] = __ldg(F.taps + e);
  const long long nout = (r.n * up + down - 1) / down;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long ja = r.j0 + tile * RS_J, jb = min(ja + RS_J, r.j0 + r.cnt);
    const long long la = max(ja, 0LL), lb = min(jb, nout);                 // outputs with inputs: [la, lb)
    long long lo = 0, hi = 0;                                              // their input span [lo, hi)
    if (la < lb) {
      lo = (la * down + half_len) / up - K + 1;
      hi = ((lb - 1) * down + half_len) / up + 1;
    }
    float acc[RS_R];
    int top[RS_R], ph[RS_R];                                               // input q - lo, tap row offset; top < 0: output is 0
#pragma unroll
    for (int k = 0; k < RS_R; k++) {
      const long long j = ja + threadIdx.x + k * RS_THREADS;
      acc[k] = 0.f;
      top[k] = -1;
      ph[k] = 0;
      if (j >= la && j < lb) {
        const long long s = j * down + half_len, q = s / up;
        top[k] = (int)(q - lo);
        ph[k] = (int)(s - q * up) * Kp;
      }
    }
    for (long long c0 = lo; c0 < hi; c0 += chunk) {
      const int cn = (int)min((long long)chunk, hi - c0), base = (int)(c0 - lo);
      __syncthreads();                                                     // the taps are written; the last pass's reads are done
      for (int e = threadIdx.x; e < cn; e += RS_THREADS) xs[e] = rs_input(r, c0 + e);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < RS_R; k++) {
        if (top[k] < 0) continue;
        const int t = top[k] - base;                                       // input q relative to the pass
        const int first = max(t - K + 1, 0), last = min(t, cn - 1);
        const float* w = taps + ph[k] + t;
        for (int e = first; e <= last; e++) acc[k] = fmaf(xs[e], w[-e], acc[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < RS_R; k++) {
      const long long j = ja + threadIdx.x + k * RS_THREADS;
      if (j >= jb) break;
      const float v = top[k] >= 0 ? acc[k] : 0.f;
      const long long o = j - r.j0;
      if (r.enc == FS2_RESAMPLE_F32) {
        static_cast<float*>(r.y)[o] = v;
      } else {
        const short pcm = pcm16_sample(v, P.scale);
        if (r.enc == FS2_RESAMPLE_PCM16) static_cast<short*>(r.y)[o] = pcm;
        else static_cast<unsigned char*>(r.y)[o] = r.enc == FS2_RESAMPLE_ULAW ? ulaw_byte(pcm) : alaw_byte(pcm);
      }
    }
  }
}

static long long rs_nout(long long n, int up, int down) { return (n * up + down - 1) / down; }

static int rs_gcd(int a, int b) { return b ? rs_gcd(b, a % b) : a; }

// The ratio and tap-table rules of include/fs2b200.h; fills one filter of the kernel.  The identity (up == down == 1, K == 1: output j
// is input j) only where the caller allows it.
static int rs_filter(int up, int down, int K, const float* taps, bool identity_ok, RsFilter& F) {
  if (!taps) return FS2_ERR_ARG;
  const bool identity = up == 1 && down == 1;
  if (identity && !(identity_ok && K == 1)) return FS2_ERR_ARG;
  if (up < 1 || down < 1 || up > FS2_RESAMPLE_MAX_FACTOR || down > FS2_RESAMPLE_MAX_FACTOR || rs_gcd(up, down) != 1) return FS2_ERR_ARG;
  const int half_len = identity ? 0 : 10 * (up > down ? up : down);
  if (!identity && K != (2 * half_len + 1 + up - 1) / up) return FS2_ERR_ARG;
  F.up = up; F.down = down; F.K = K; F.Kp = K | 1; F.half_len = half_len; F.taps = taps;
  const long long span = ((long long)(RS_J - 1) * down + up - 1) / up + K + 1;
  F.chunk = (int)(span < RS_CHUNK_MAX ? span : RS_CHUNK_MAX);
  return FS2_OK;
}

// The offline, window and streams calls: one filter, one encoding for every row.
static int rs_single(int up, int down, int K, const float* taps, float scale, int pcm16, RsParams& P) {
  P = RsParams{};
  FS2_TRY(rs_filter(up, down, K, taps, false, P.f[0]));
  P.n_filters = 1;
  P.enc = pcm16 ? FS2_RESAMPLE_PCM16 : FS2_RESAMPLE_F32; P.scale = scale;
  return FS2_OK;
}

static cudaError_t rs_setup() {
  int dev = 0, mx = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&mx, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return e == cudaSuccess ? cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mx) : e;
}

// Launches B rows of at most max_cnt outputs each, about four blocks per SM in all, with the shared memory of the largest filter.
static int rs_launch(const RsParams& P, int B, long long max_cnt, cudaStream_t s) {
  size_t smem = 0;
  int K_max = 0;
  for (int i = 0; i < P.n_filters; i++) {
    smem = std::max(smem, ((size_t)P.f[i].up * P.f[i].Kp + P.f[i].chunk) * sizeof(float));
    K_max = std::max(K_max, P.f[i].K);
  }
  int derr = FS2_OK, dev = 0, mx = 0;
  DevState* dv = dev_state(&derr);
  if (!dv) return derr;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&mx, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e != cudaSuccess) return FS2_ERR_CUDA - (int)e;
  if (smem > (size_t)mx) return FS2_ERR_UNSUPPORTED;
  FS2_TRY(dev_once(dv->resample_ready, rs_setup));
  const long long tiles = (max_cnt + RS_J - 1) / RS_J, want = (4LL * dv->num_sms.load() + B - 1) / B;
  const unsigned gx = (unsigned)(tiles < want ? tiles : want);
  prof_before(s);
  resample_kernel<<<dim3(gx, (unsigned)B), RS_THREADS, smem, s>>>(P);
  FS2_LAUNCH_CHECK();
  prof_after(s, 3, 2.0 * (double)B * (double)max_cnt * K_max);
  return FS2_OK;
}

static int resample_window(const fs2_resample_window_args* a, cudaStream_t s) {
  if (!a || a->B < 1 || a->B > 65535 || a->N < 1 || !a->y) return FS2_ERR_ARG;
  RsParams P;
  FS2_TRY(rs_single(a->up, a->down, a->K, a->taps, a->scale, a->pcm16, P));
  const long long nout = rs_nout(a->N, a->up, a->down), cnt = a->j1 - a->j0;
  if (a->j0 < 0 || cnt < 1 || a->j1 > nout || (a->B > 1 && a->y_batch_stride < cnt)) return FS2_ERR_ARG;
  if (a->i0 > a->i1 || a->i1 > a->i2 || (a->i1 > a->i0 && !a->x0) || (a->i2 > a->i1 && !a->x1)) return FS2_ERR_ARG;
  if (a->lens && a->lens_scale < 1) return FS2_ERR_ARG;
  // every input of [0, N) that outputs [j0, j1) read must have been given
  const long long lo = std::max<long long>((a->j0 * a->down + P.f[0].half_len) / a->up - a->K + 1, 0);
  const long long hi = std::min<long long>(((a->j1 - 1) * a->down + P.f[0].half_len) / a->up + 1, a->N);
  if (lo < hi && (lo < a->i0 || hi > a->i2)) return FS2_ERR_ARG;
  P.x0 = a->x0; P.x0_bs = a->x0_batch_stride;
  P.x1 = a->x1; P.x1_bs = a->x1_batch_stride;
  P.i0 = a->i0; P.i1 = a->i1; P.i2 = a->i2; P.N = a->N;
  P.lens = a->lens; P.lens_scale = a->lens_scale;
  P.j0 = a->j0; P.j1 = a->j1;
  P.y = a->y; P.y_bs = a->y_batch_stride;
  return rs_launch(P, a->B, cnt, s);
}

}  // namespace fs2

using namespace fs2;

static_assert(sizeof(fs2_resample_args) == 88, "fs2_resample_args layout is pinned by the binding");
static_assert(sizeof(fs2_resample_window_args) == 144, "fs2_resample_window_args layout is pinned by the binding");
static_assert(sizeof(fs2_resample_stream_t) == 64, "fs2_resample_stream_t layout is pinned by the binding");
static_assert(sizeof(fs2_resample_streams_args) == 64, "fs2_resample_streams_args layout is pinned by the binding");
static_assert(sizeof(fs2_resample_filter_t) == 24, "fs2_resample_filter_t layout is pinned by the binding");
static_assert(sizeof(fs2_resample_mixed_stream_t) == 80, "fs2_resample_mixed_stream_t layout is pinned by the binding");
static_assert(sizeof(fs2_resample_mixed_args) == 232, "fs2_resample_mixed_args layout is pinned by the binding");

extern "C" {

int fs2_resample(const fs2_resample_args* a, fs2_stream_t st) {
  if (!a || a->N < 1 || !a->x) return FS2_ERR_ARG;
  if (a->up < 1 || a->down < 1) return FS2_ERR_ARG;
  fs2_resample_window_args w{};
  w.B = a->B; w.up = a->up; w.down = a->down; w.K = a->K; w.taps = a->taps;
  w.x0 = a->x; w.x0_batch_stride = a->x_batch_stride;
  w.i0 = 0; w.i1 = a->N; w.i2 = a->N; w.N = a->N;
  w.lens = a->lens; w.lens_scale = a->lens_scale;
  w.j0 = 0; w.j1 = rs_nout(a->N, a->up, a->down);
  w.y = a->y; w.y_batch_stride = a->y_batch_stride;
  w.pcm16 = a->pcm16; w.scale = a->scale;
  return resample_window(&w, (cudaStream_t)st);
}

int fs2_resample_window(const fs2_resample_window_args* a, fs2_stream_t st) { return resample_window(a, (cudaStream_t)st); }

int fs2_resample_streams(const fs2_resample_streams_args* a, fs2_stream_t st) {
  if (!a || a->B < 1 || a->B > 65535 || !a->table || a->max_out < 1 || !a->y || (a->B > 1 && a->y_batch_stride < a->max_out))
    return FS2_ERR_ARG;
  RsParams P;
  FS2_TRY(rs_single(a->up, a->down, a->K, a->taps, a->scale, a->pcm16, P));
  P.table = a->table; P.max_out = a->max_out;
  P.y = a->y; P.y_bs = a->y_batch_stride;
  return rs_launch(P, a->B, a->max_out, (cudaStream_t)st);
}

int fs2_resample_streams_mixed(const fs2_resample_mixed_args* a, fs2_stream_t st) {
  if (!a || a->B < 1 || a->B > 65535 || !a->table || a->max_out < 1 || !a->y || !aligned16(a->y)) return FS2_ERR_ARG;
  if (a->n_filters < 1 || a->n_filters > FS2_RESAMPLE_MAX_FILTERS) return FS2_ERR_ARG;
  RsParams P{};
  for (int i = 0; i < a->n_filters; i++) {
    const fs2_resample_filter_t& f = a->filters[i];
    FS2_TRY(rs_filter(f.up, f.down, f.K, f.taps, true, P.f[i]));
  }
  P.n_filters = a->n_filters; P.scale = a->scale;
  P.mixed = a->table; P.max_out = a->max_out;
  P.y = a->y;
  return rs_launch(P, a->B, a->max_out, (cudaStream_t)st);
}

}  // extern "C"
