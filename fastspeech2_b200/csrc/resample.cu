// Polyphase FIR sample-rate conversion of the waveform: scipy.signal.resample_poly's arithmetic in fp32 (include/fs2b200.h).
// One kernel serves the offline, window and streams calls; they differ only in where a row's input pieces, length and output range
// come from (RsRow).
#include <algorithm>
#include <cstddef>

#include "common.cuh"

namespace fs2 {

constexpr int RS_THREADS = 256, RS_R = 8, RS_J = RS_THREADS * RS_R;   // outputs per tile: RS_R per thread
constexpr int RS_CHUNK_MAX = 8192;                                     // input floats staged per pass

// One row: input samples [i0, i1) at x0, [i1, i2) at x1, n samples in all (inputs outside [0, n) are zero); outputs [j0, j0 + cnt)
// go to y[j - j0].
struct RsRow {
  const float *x0, *x1;
  long long i0, i1, i2, n, j0, cnt;
  void* y;
};

struct RsParams {
  int up, down, K, Kp, half_len, chunk;
  const float* taps;
  int pcm16; float scale;
  // offline and window calls: pieces shared by every row, with batch strides
  const float *x0, *x1; long long x0_bs, x1_bs, i0, i1, i2, N, j0, j1;
  const int32_t* lens; int lens_scale;
  void* y; long long y_bs;
  // streams call: a device record per row
  const fs2_resample_stream_t* table; long long max_out;
};

__device__ __forceinline__ RsRow rs_row(const RsParams& P, int b) {
  RsRow r;
  const size_t ob = (size_t)b * P.y_bs * (P.pcm16 ? sizeof(short) : sizeof(float));
  r.y = static_cast<char*>(P.y) + ob;
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

// grid (tiles, rows).  Each block copies the [up][K] taps to shared memory once (row stride Kp = K | 1, odd, so that the phases of a
// warp's 32 consecutive outputs spread over the banks) and then walks its row's tiles of RS_J outputs.  Per tile it stages the input
// span of the tile's outputs in shared memory, in passes of at most `chunk` samples, so that adjacent outputs share their input loads
// from global memory; thread t owns outputs t + 256 r (r < RS_R), so loads, stores and tap reads of a warp are consecutive.  Each
// output accumulates its taps in ascending input order across the passes.
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const RsParams P) {
  extern __shared__ float smem[];
  float* taps = smem;
  float* xs = smem + P.up * P.Kp;
  const RsRow r = rs_row(P, blockIdx.y);
  const long long n_tiles = (r.cnt + RS_J - 1) / RS_J;
  if ((long long)blockIdx.x >= n_tiles) return;
  for (int e = threadIdx.x; e < P.up * P.K; e += RS_THREADS) taps[(e / P.K) * P.Kp + e % P.K] = __ldg(P.taps + e);
  const long long nout = (r.n * P.up + P.down - 1) / P.down;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long ja = r.j0 + tile * RS_J, jb = min(ja + RS_J, r.j0 + r.cnt);
    const long long la = max(ja, 0LL), lb = min(jb, nout);                 // outputs with inputs: [la, lb)
    long long lo = 0, hi = 0;                                              // their input span [lo, hi)
    if (la < lb) {
      lo = (la * P.down + P.half_len) / P.up - P.K + 1;
      hi = ((lb - 1) * P.down + P.half_len) / P.up + 1;
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
        const long long s = j * P.down + P.half_len, q = s / P.up;
        top[k] = (int)(q - lo);
        ph[k] = (int)(s - q * P.up) * P.Kp;
      }
    }
    for (long long c0 = lo; c0 < hi; c0 += P.chunk) {
      const int cn = (int)min((long long)P.chunk, hi - c0), base = (int)(c0 - lo);
      __syncthreads();                                                     // the taps are written; the last pass's reads are done
      for (int e = threadIdx.x; e < cn; e += RS_THREADS) xs[e] = rs_input(r, c0 + e);
      __syncthreads();
#pragma unroll
      for (int k = 0; k < RS_R; k++) {
        if (top[k] < 0) continue;
        const int t = top[k] - base;                                       // input q relative to the pass
        const int first = max(t - P.K + 1, 0), last = min(t, cn - 1);
        const float* w = taps + ph[k] + t;
        for (int e = first; e <= last; e++) acc[k] = fmaf(xs[e], w[-e], acc[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < RS_R; k++) {
      const long long j = ja + threadIdx.x + k * RS_THREADS;
      if (j >= jb) break;
      const float v = top[k] >= 0 ? acc[k] : 0.f;
      if (P.pcm16) static_cast<short*>(r.y)[j - r.j0] = pcm16_sample(v, P.scale);
      else static_cast<float*>(r.y)[j - r.j0] = v;
    }
  }
}

static long long rs_nout(long long n, int up, int down) { return (n * up + down - 1) / down; }

static int rs_gcd(int a, int b) { return b ? rs_gcd(b, a % b) : a; }

// The ratio and tap-table rules of include/fs2b200.h; fills the kernel's filter fields.
static int rs_filter(int up, int down, int K, const float* taps, float scale, int pcm16, RsParams& P) {
  if (up < 1 || down < 1 || (up == 1 && down == 1) || up > FS2_RESAMPLE_MAX_FACTOR || down > FS2_RESAMPLE_MAX_FACTOR) return FS2_ERR_ARG;
  if (rs_gcd(up, down) != 1 || !taps) return FS2_ERR_ARG;
  const int half_len = 10 * (up > down ? up : down);
  if (K != (2 * half_len + 1 + up - 1) / up) return FS2_ERR_ARG;
  P = RsParams{};
  P.up = up; P.down = down; P.K = K; P.Kp = K | 1; P.half_len = half_len; P.taps = taps;
  P.pcm16 = pcm16 ? 1 : 0; P.scale = scale;
  const long long span = ((long long)(RS_J - 1) * down + up - 1) / up + K + 1;
  P.chunk = (int)(span < RS_CHUNK_MAX ? span : RS_CHUNK_MAX);
  return FS2_OK;
}

static cudaError_t rs_setup() {
  int dev = 0, mx = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&mx, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return e == cudaSuccess ? cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, mx) : e;
}

// Launches B rows of at most max_cnt outputs each, about four blocks per SM in all.
static int rs_launch(const RsParams& P, int B, long long max_cnt, cudaStream_t s) {
  const size_t smem = ((size_t)P.up * P.Kp + P.chunk) * sizeof(float);
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
  prof_after(s, 3, 2.0 * (double)B * (double)max_cnt * P.K);
  return FS2_OK;
}

static int resample_window(const fs2_resample_window_args* a, cudaStream_t s) {
  if (!a || a->B < 1 || a->B > 65535 || a->N < 1 || !a->y) return FS2_ERR_ARG;
  RsParams P;
  FS2_TRY(rs_filter(a->up, a->down, a->K, a->taps, a->scale, a->pcm16, P));
  const long long nout = rs_nout(a->N, a->up, a->down), cnt = a->j1 - a->j0;
  if (a->j0 < 0 || cnt < 1 || a->j1 > nout || (a->B > 1 && a->y_batch_stride < cnt)) return FS2_ERR_ARG;
  if (a->i0 > a->i1 || a->i1 > a->i2 || (a->i1 > a->i0 && !a->x0) || (a->i2 > a->i1 && !a->x1)) return FS2_ERR_ARG;
  if (a->lens && a->lens_scale < 1) return FS2_ERR_ARG;
  // every input of [0, N) that outputs [j0, j1) read must have been given
  const long long lo = std::max<long long>((a->j0 * a->down + P.half_len) / a->up - a->K + 1, 0);
  const long long hi = std::min<long long>(((a->j1 - 1) * a->down + P.half_len) / a->up + 1, a->N);
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
  FS2_TRY(rs_filter(a->up, a->down, a->K, a->taps, a->scale, a->pcm16, P));
  P.table = a->table; P.max_out = a->max_out;
  P.y = a->y; P.y_bs = a->y_batch_stride;
  return rs_launch(P, a->B, a->max_out, (cudaStream_t)st);
}

}  // extern "C"
