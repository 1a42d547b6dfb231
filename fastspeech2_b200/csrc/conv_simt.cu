// fp32 CUDA-core implicit-GEMM Conv1d over channels-last activations.
//
// This is the exact-precision path (plain fp32 FMA, fp32 accumulate): it serves every layer upstream of the
// discrete duration / pitch-bucket decisions, where the parity budget is ~1e-6 (SURVEY.md section 7, hard part 2),
// and is the fallback for shapes the tensor-core path does not take.  One kernel covers nn.Linear (taps = 1),
// nn.Conv1d with dilation, and a phase group of ConvTranspose1d (see fs2b200.h).
//
// Tiling: CTA = 128 (or 64, for small problems) rows (time) x BN output channels, BK = 16, 256 threads, TM x TN register tile per thread,
// A tile transposed into smem so the inner product reads two broadcast float4 (A) and two conflict-free float4 (B)
// per 64 FMAs; global->register->smem double buffering, one __syncthreads per k-step.
#include "common.cuh"

namespace fs2 {

constexpr int BK = 16;

struct ConvP {
  const float* x; long long xbs, xrs;
  int B, T, Cin;
  const float* w; const float* bias;
  int N, taps, dil, pad;
  int in_act; float in_slope;
  int out_act; float out_slope;
  const float* res; long long rbs, rrs;
  float alpha; int accumulate;
  const int* row_lens;
  float* y; long long ybs, yrs;
  int tiles_per_batch;
  const int* x_lens; int lens_scale;   // ragged batch (fs2_conv1d_args::x_lens) or NULL
};

template <int BM, int BN, int ACT>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvP p) {
  constexpr int AS_LD = BM + 4;
  constexpr int TM = BM / 16;              // 8 or 4 rows per thread
  constexpr int A_PER_THREAD = BM * BK / 4 / 256;   // float4 loads of the A tile per thread (2 or 1)
  constexpr int TN = BN / 16;              // 8, 4 or 2 columns per thread
  constexpr int NG = (TN == 8) ? 2 : 1;    // column groups per thread
  constexpr int GW = (TN == 2) ? 2 : 4;    // group width
  constexpr int B_F4 = BK * BN / 4;        // float4 per B tile
  constexpr int B_PER_THREAD = (B_F4 + 255) / 256;

  __shared__ __align__(16) float As[2][BK][AS_LD];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.x / p.tiles_per_batch;
  const int t0 = (blockIdx.x % p.tiles_per_batch) * BM;
  const int n0 = blockIdx.y * BN;
  // ragged batch: input rows t >= n_b read as zero, and a tile lying wholly at or beyond n_b has nothing to compute (its rows are unspecified)
  const int tend = p.x_lens ? ragged_rows(p.x_lens, p.lens_scale, p.T, b) : p.T;
  if (t0 >= tend) return;

  const float* xb = p.x + (long long)b * p.xbs;
  const int kc = p.Cin / BK;               // k-steps per tap
  const int KT = p.taps * kc;

  float acc[TM][NG * GW];
#pragma unroll
  for (int i = 0; i < TM; i++)
#pragma unroll
    for (int j = 0; j < NG * GW; j++) acc[i][j] = 0.f;

  float4 ra[A_PER_THREAD];
  float4 rb[B_PER_THREAD];

  auto load_global = [&](int kt) {
    const int tap = kt / kc;
    const int c0 = (kt - tap * kc) * BK;
    const int shift = tap * p.dil - p.pad;
#pragma unroll
    for (int i = 0; i < A_PER_THREAD; i++) {
      const int f = tid + i * 256;
      const int row = f >> 2, c4 = f & 3;
      const int t = t0 + row + shift;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (t >= 0 && t < tend) {
        v = __ldg(reinterpret_cast<const float4*>(xb + (long long)t * p.xrs + c0 + c4 * 4));
        if (p.in_act == FS2_ACT_LRELU) {
          v.x = v.x > 0.f ? v.x : v.x * p.in_slope;
          v.y = v.y > 0.f ? v.y : v.y * p.in_slope;
          v.z = v.z > 0.f ? v.z : v.z * p.in_slope;
          v.w = v.w > 0.f ? v.w : v.w * p.in_slope;
        }
      }
      ra[i] = v;
    }
    const float* wt = p.w + ((long long)tap * p.Cin + c0) * p.N;
#pragma unroll
    for (int i = 0; i < B_PER_THREAD; i++) {
      const int f = tid + i * 256;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f < B_F4) {
        const int k = f / (BN / 4), n4 = f % (BN / 4);
        const int n = n0 + n4 * 4;
        if (n < p.N) v = __ldg(reinterpret_cast<const float4*>(wt + (long long)k * p.N + n));
      }
      rb[i] = v;
    }
  };
  auto store_smem = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_PER_THREAD; i++) {
      const int f = tid + i * 256;
      const int row = f >> 2, c4 = f & 3;
      As[buf][c4 * 4 + 0][row] = ra[i].x;
      As[buf][c4 * 4 + 1][row] = ra[i].y;
      As[buf][c4 * 4 + 2][row] = ra[i].z;
      As[buf][c4 * 4 + 3][row] = ra[i].w;
    }
#pragma unroll
    for (int i = 0; i < B_PER_THREAD; i++) {
      const int f = tid + i * 256;
      if (f < B_F4) {
        const int k = f / (BN / 4), n4 = f % (BN / 4);
        *reinterpret_cast<float4*>(&Bs[buf][k][n4 * 4]) = rb[i];
      }
    }
  };

  load_global(0);
  store_smem(0);
  __syncthreads();

  for (int kt = 0; kt < KT; kt++) {
    const int buf = kt & 1;
    if (kt + 1 < KT) load_global(kt + 1);
#pragma unroll
    for (int k = 0; k < BK; k++) {
      float av[TM];
      {
        const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
        av[0] = a0.x; av[1] = a0.y; av[2] = a0.z; av[3] = a0.w;
        if constexpr (TM == 8) {
          const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
          av[4] = a1.x; av[5] = a1.y; av[6] = a1.z; av[7] = a1.w;
        }
      }
      float bv[NG * GW];
      if constexpr (TN == 2) {
        const float2 b0 = *reinterpret_cast<const float2*>(&Bs[buf][k][tx * 2]);
        bv[0] = b0.x; bv[1] = b0.y;
      } else {
        const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
        bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w;
        if constexpr (TN == 8) {
          const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][BN / 2 + tx * 4]);
          bv[4] = b1.x; bv[5] = b1.y; bv[6] = b1.z; bv[7] = b1.w;
        }
      }
#pragma unroll
      for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < NG * GW; j++) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < KT) store_smem(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue: bias, activation, residual, alpha/accumulate, row mask ----
  const int len_b = p.row_lens ? p.row_lens[b] : p.T;
#pragma unroll
  for (int i = 0; i < TM; i++) {
    const int m = (i < 4) ? (ty * 4 + i) : (64 + ty * 4 + (i - 4));
    const int t = t0 + m;
    if (t >= p.T) continue;
    float* yrow = p.y + (long long)b * p.ybs + (long long)t * p.yrs;
    const float* rrow = p.res ? (p.res + (long long)b * p.rbs + (long long)t * p.rrs) : nullptr;
    const bool dead = t >= len_b;
#pragma unroll
    for (int g = 0; g < NG; g++) {
      const int nb = n0 + ((TN == 2) ? tx * 2 : (g * (BN / 2) + tx * 4));
      if (nb >= p.N) continue;
      float v[GW];
#pragma unroll
      for (int j = 0; j < GW; j++) {
        float u = acc[i][g * GW + j] + (p.bias ? __ldg(p.bias + nb + j) : 0.f);
        u = ACT == FS2_ACT_RELU ? fmaxf(u, 0.f) : ACT == FS2_ACT_TANH ? tanhf(u) : ACT == FS2_ACT_LRELU ? (u > 0.f ? u : u * p.out_slope) : u;
        if (rrow) u += rrow[nb + j];
        u *= p.alpha;
        if (p.accumulate) u += yrow[nb + j];
        v[j] = dead ? 0.f : u;
      }
      if constexpr (GW == 4) {
        *reinterpret_cast<float4*>(yrow + nb) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
        *reinterpret_cast<float2*>(yrow + nb) = make_float2(v[0], v[1]);
      }
    }
  }
}

int conv1d_simt(const fs2_conv1d_args* a, cudaStream_t s) {
  if (!a || !a->x || !a->w || !a->y) return FS2_ERR_ARG;
  if (a->B <= 0 || a->T <= 0 || a->Cin <= 0 || a->N <= 0 || a->taps <= 0) return FS2_ERR_ARG;
  if (a->Cin % BK != 0 || a->N % 4 != 0) return FS2_ERR_UNSUPPORTED;
  if ((a->x_row_stride & 3) || (a->x_batch_stride & 3) || (a->y_row_stride & 3) || (a->y_batch_stride & 3)) return FS2_ERR_UNSUPPORTED;
  if (a->res && ((a->res_row_stride & 3) || (a->res_batch_stride & 3))) return FS2_ERR_UNSUPPORTED;
  if (!aligned16(a->x) || !aligned16(a->w) || !aligned16(a->y) || (a->res && !aligned16(a->res))) return FS2_ERR_ARG;
  if (a->in_act != FS2_ACT_NONE && a->in_act != FS2_ACT_LRELU) return FS2_ERR_UNSUPPORTED;
  ConvP p;
  p.x = a->x; p.xbs = a->x_batch_stride; p.xrs = a->x_row_stride;
  p.B = a->B; p.T = a->T; p.Cin = a->Cin;
  p.w = a->w; p.bias = a->bias;
  p.N = a->N; p.taps = a->taps; p.dil = a->dilation; p.pad = a->pad_left;
  p.in_act = a->in_act; p.in_slope = a->in_slope;
  p.out_act = a->out_act; p.out_slope = a->out_slope;
  p.res = a->res; p.rbs = a->res_batch_stride; p.rrs = a->res_row_stride;
  p.alpha = a->alpha; p.accumulate = a->accumulate;
  p.row_lens = a->row_lens;
  p.x_lens = a->x_lens; p.lens_scale = a->lens_scale;
  p.y = a->y; p.ybs = a->y_batch_stride; p.yrs = a->y_row_stride;
  int derr = FS2_OK;
  DevState* dv = dev_state(&derr);                      // SM count of the current device
  if (!dv) return derr;
  const long long num_sms = dv->num_sms.load(std::memory_order_relaxed);
  // 128-row tiles by default; 64-row tiles when the grid would not even give every SM two CTAs (encoder / predictors: 2048 rows)
  const int nblk = a->N > 64 ? (a->N + 127) / 128 : 1;
  const bool small = (long long)((a->T + 127) / 128) * a->B * nblk < 2LL * num_sms;
  const int bm = small ? 64 : 128;
  p.tiles_per_batch = (a->T + bm - 1) / bm;
  const long long gx = (long long)p.tiles_per_batch * a->B;
  if (gx > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
  prof_before(s);
#define FS2_SIMT_ACT(BM_, BN_, grid_)                                                                      \
  switch (a->out_act) {                                                                                    \
    case FS2_ACT_RELU: conv_simt_kernel<BM_, BN_, FS2_ACT_RELU><<<grid_, 256, 0, s>>>(p); break;           \
    case FS2_ACT_TANH: conv_simt_kernel<BM_, BN_, FS2_ACT_TANH><<<grid_, 256, 0, s>>>(p); break;           \
    case FS2_ACT_LRELU: conv_simt_kernel<BM_, BN_, FS2_ACT_LRELU><<<grid_, 256, 0, s>>>(p); break;         \
    default: conv_simt_kernel<BM_, BN_, FS2_ACT_NONE><<<grid_, 256, 0, s>>>(p); break;                     \
  }
#define FS2_SIMT_LAUNCH(BN_, grid_)                   \
  if (small) { FS2_SIMT_ACT(64, BN_, grid_) } else { FS2_SIMT_ACT(128, BN_, grid_) }
  // narrow outputs on small problems (FFN w_2, predictor convs: 2048 rows x 256 channels): 64-column CTAs double the CTA count
  // while the 128-column grid leaves SMs idle
  const bool narrow_small = small && a->N > 64 && (long long)gx * ((a->N + 127) / 128) < num_sms;
  if (a->N > 64 && !narrow_small) {
    dim3 grid((unsigned)gx, (a->N + 127) / 128);
    FS2_SIMT_LAUNCH(128, grid)
  } else if (a->N > 32) {
    dim3 grid((unsigned)gx, (a->N + 63) / 64);
    FS2_SIMT_LAUNCH(64, grid)
  } else {
    dim3 grid((unsigned)gx, 1);
    FS2_SIMT_LAUNCH(32, grid)
  }
#undef FS2_SIMT_LAUNCH
#undef FS2_SIMT_ACT
  prof_after(s, 4, 2.0 * a->B * a->T * (double)a->Cin * a->taps * a->N);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
