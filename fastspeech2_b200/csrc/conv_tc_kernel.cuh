// [device code; host side and heuristics: conv_tc.cu]
// wgmma (Hopper warpgroup MMA) implicit-GEMM Conv1d over channels-last activations, error-compensated split-FP16.
//
//   y[b,t,n] = epilogue( sum_{tap} sum_c act(x[b, t + tap*dil - pad, c]) * w[tap][c][n] )        (contract: fs2_conv1d)
//
// Why a split: single-pass TF32 / FP16 / BF16 operands miss the parity bars (mel 1.2e-3 vs 1e-3, waveform 5.3e-4 vs 1e-4,
// SURVEY.md section 7).  Each fp32 operand is split x = hi + lo with hi = fp16(x), lo = fp16(x - hi) (x - hi is exact in
// fp32): 22 significant bits, the same as a TF32 hi/lo split, but FP16 MMAs have K = 16 per instruction -- twice the
// FLOPs per instruction and per shared-memory byte of TF32.  D += A_lo*B_hi + A_hi*B_hi + A_hi*B_lo, fp32 accumulate in
// registers.  Weights are pre-scaled by a per-layer power of two (kept in a 128-byte header of the tiled buffer) so that their lo
// parts stay in fp16's normal range; activations are used unscaled (|x| > 65504 saturates in the convert; a lo part below 2^-14 only costs an
// ABSOLUTE error < 3e-8).  Emulated end to end on the CPU (exact accumulation) this split is as accurate as fp32 convolution
// on both the synthetic and the shipped HiFi-GAN checkpoint; on the GPU the tensor core's truncating accumulator is what remains.
//
// Persistent, warp-specialised kernel: one CTA per SM walks a list of work items (one 128-row time tile of one utterance x one
// block of NB <= 128 output channels); three roles overlap through mbarrier rings:
//   warp 8      weight producer: every (tap, 16-channel K-block) weight stage is ONE cp.async.bulk (TMA bulk engine) of a
//               host-pre-split, host-pre-tiled smem image  [hi|lo][16-byte K-chunk][n][8 halfs].
//   warps 9-16  activation transform: read the [128 + (taps-1)*dil] x 16-channel slab of a K-block ONCE from global
//               (one 32-byte sector per row and 8 channels, a register ring of K-blocks in flight), apply the input activation,
//               split hi/lo and store both in the no-swizzle K-major layout [16-byte K-chunk][row][8 halfs].  There a core
//               matrix (8 rows x 16 B) starting at ANY row is 128 contiguous bytes, so each conv tap is just the same slab with
//               the descriptor start address advanced by tap*dil rows: the slab is loaded and split once per K-block, not once per tap.
//   warps 0-7   two consumer warpgroups, 64 output rows each: per weight stage 3 (split terms) wgmma m64nNBk16 with register
//               accumulators (or one FP16 + one E4M3 K = 32 MMA, TcP::f8), then the epilogue straight from the accumulator
//               fragments: bias / activation / residual / alpha / accumulate / pad-row mask -> global stores.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace fs2 {

constexpr int TC_KB = 16;          // input channels per K-block (one K=16 FP16 MMA per split term)
constexpr int TC_CHUNKS = TC_KB / 8;  // 16-byte K-chunks (8 halfs) per K-block
constexpr int TC_SA_MAX = 8;       // activation slab stages (runtime p.SA)
constexpr int TC_SB_MAX = 8;       // weight stages (runtime p.SB)
constexpr int TC_TW = 8;            // transform warps
constexpr int TC_TTHREADS = TC_TW * 32;
constexpr int TC_CWG = 2;          // consumer warpgroups (64 output rows each)
constexpr int TC_CTHREADS = TC_CWG * 128;
constexpr int TC_THREADS = TC_CTHREADS + 32 + TC_TTHREADS;   // consumer warpgroups, producer warp, transform warps
constexpr int TC_DEPTH = 2;         // K-blocks of activation loads in flight per transform thread (register ring)
constexpr int TC_LD = 3;           // (row, K-chunk) items (2 float4 loads each) per transform thread per K-block: 256 * 3 / 2 >= 384 rows
constexpr int TC_HDR = 128;        // bytes of header in front of the weight tiles: float[0] = 1 / weight scale

struct TcP {
  const float* x; long long xbs, xrs;
  int B, T, Cin;
  const float* wt;                 // tiled weights, see packing.pack_conv_tc
  const float* bias;
  int N;                           // total output channels
  int NB;                          // output channels per work item (MMA N), N % NB == 0, NB % 16 == 0, NB <= 128
  int taps, dil, pad;
  int in_act; float in_slope;
  int out_act; float out_slope;
  const float* res; long long rbs, rrs;
  float alpha; int accumulate;
  const int* row_lens;
  float* y; long long ybs, yrs;
  int TG;                          // accumulators per tile: 1 = all split terms together, 2 = {hi*hi | the two cross terms}
  int SA, SB;                      // ring depths
  int TPS;                         // conv taps per weight stage (small NB: several taps share one bulk copy / one handshake)
  int R;                           // slab rows held in smem (>= 128 + (taps-1)*dil, R % 8 == 4)
  int tiles_per_batch;             // work items per utterance
  int n_items;                     // total work items = (N/NB) * B * tiles_per_batch
  int nseg;                        // K-segments per output tile (1 = plain conv).  > 1: the conv is the sum of nseg one-tap slices over p.Cin (= 256)
                                   // input channels each, slice s = (tap = s / seg_nkc, channel chunk = s % seg_nkc); every slice is its own work unit with a
                                   // fresh accumulator, and the units of one tile run back to back on one CTA, adding into y in fp32 (FS2_TC_VARIANT_SEGMENTED)
  int seg_nkc;                     // channel chunks per tap
  long long seg_wbytes;            // bytes between the tile buffers of consecutive slices
  int f8;                          // operand split: 0 = three FP16 MMAs (hi*hi + lo*hi + hi*lo), 1 = FP16 main term + ONE E4M3 (K = 32) correction MMA
  const int* x_lens;               // ragged batch (fs2_conv1d_args::x_lens) or NULL; n_items / tiles_per_batch then only bound the grid
  int lens_scale;
};

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// 8 consecutive floats (one 32-byte sector) as two 128-bit read-only loads
__device__ __forceinline__ void ldg256(float (&d)[8], const float* src) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src) + 1);
  d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
}
// fp16x2 {lo = a0, hi = a1}, round-to-nearest, |x| > 65504 saturates instead of becoming inf: SASS F2FP.SATFINITE.F16.F32.PACK_AB
__device__ __forceinline__ uint32_t cvt_f16x2_sat(float a0, float a1) {
  uint32_t h;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(a1), "f"(a0));
  return h;
}

// e4m3x2 {byte 0 = a0, byte 1 = a1}, round-to-nearest, saturating at +-448
__device__ __forceinline__ uint32_t cvt_e4m3x2_sat(float a0, float a1) {
  unsigned short h;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(h) : "f"(a1), "f"(a0));
  return (uint32_t)h;
}

// mbarrier ring cursor without runtime div/mod (an integer division per tap was on the MMA issuer's critical path)
struct Ring {
  uint32_t idx = 0, phase = 0;
  __device__ __forceinline__ void advance(uint32_t n) {
    if (++idx == n) { idx = 0; phase ^= 1u; }
  }
};

struct Item { int nblk, b, t0; };
__device__ __forceinline__ Item decode_item(const TcP& p, int item) {
  const int per_blk = p.B * p.tiles_per_batch;
  Item it;
  it.nblk = item / per_blk;
  const int rem = item - it.nblk * per_blk;
  it.b = rem / p.tiles_per_batch;
  it.t0 = (rem - it.b * p.tiles_per_batch) * 128;
  return it;
}

// Ragged batch (TcP::x_lens, RsP::lens): utterance b has n_b = ragged_rows(...) rows, and the work items of one channel block are the
// live `tile`-row tiles of utterance 0, 1, ... back to back: sum_b ceil(n_b / tile) of them, so no tile lying wholly in the padding is
// ever scheduled.
// Monotone cursor over that compacted sequence.  Every role visits its items in increasing order (item = blockIdx.x, + gridDim.x, ...),
// so the cursor only moves forward and each length is loaded once per channel block: no table, no cap on B, no host sync.
// MIN_ROWS > 0: an utterance with fewer rows counts as empty (the fused attention kernel leaves those to the exact one).
template <int MIN_ROWS>
struct RaggedWalkT {
  int live;                        // live tiles per channel block
  int nblk, b, before, rows;       // cursor: channel block, utterance, live tiles of utterances < b in the block, n_b
  __device__ __forceinline__ static int rows_of(const int* lens, int scale, int cap, int b) {
    const int n = ragged_rows(lens, scale, cap, b);
    if constexpr (MIN_ROWS > 0) return n < MIN_ROWS ? 0 : n;
    return n;
  }
  __device__ __forceinline__ void init(const int* lens, int scale, int cap, int B, int tile) {
    live = 0;
    for (int i = 0; i < B; i++) live += (rows_of(lens, scale, cap, i) + tile - 1) / tile;
    nblk = 0; b = 0; before = 0; rows = rows_of(lens, scale, cap, 0);
  }
  __device__ __forceinline__ Item item(const int* lens, int scale, int cap, int tile, int i) {   // i < live * channel blocks
    const int blk = i / live, rem = i - blk * live;
    if (blk != nblk) { nblk = blk; b = 0; before = 0; rows = rows_of(lens, scale, cap, 0); }
    for (int nt = (rows + tile - 1) / tile; rem >= before + nt; nt = (rows + tile - 1) / tile) {
      before += nt;
      rows = rows_of(lens, scale, cap, ++b);
    }
    Item it;
    it.nblk = blk; it.b = b; it.t0 = (rem - before) * tile;
    return it;
  }
};
using RaggedWalk = RaggedWalkT<0>;

template <int ACT>
__device__ __forceinline__ float tc_act(float v, float slope) {
  if (ACT == FS2_ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == FS2_ACT_TANH) return tanhf(v);
  if (ACT == FS2_ACT_LRELU) return v > 0.f ? v : v * slope;
  return v;
}

// Operand scales of the f16 + f8 split (TcP::f8): activation lo * 2^12 and hi (unscaled) are rounded to E4M3; the packer stores
// weight hi * 2^-12 and lo (unscaled) in E4M3 (packing.pack_conv_tc), so both correction products carry the main term's scale.
// |x| <= 448 stays inside E4M3; beyond that the correction of that element saturates (the result degrades towards single-pass
// fp16 accuracy for it, never to garbage).
constexpr float TC_F8_LO_SCALE = 4096.f;
constexpr float TC_F8_HI_SCALE = 1.f;

// One K-block of one transform thread: input activation, operand split, stores into the slab planes.
//   F8 = false: plane 0 = fp16 hi, plane 1 = fp16 lo, both [16-byte K-chunk of 8 channels][row][8 halfs].
//   F8 = true : plane 0 = fp16 hi as above; plane 1 = E4M3 [chunk 0: lo * 2^12 of the 16 channels | chunk 1: hi of the 16 channels][row][16 bytes]
//               -- the A operand of one K = 32 E4M3 MMA whose B operand is [weight hi ; weight lo].
template <bool LRELU, bool F8, int LD>
__device__ __forceinline__ void tc_convert_store(const float (&src)[LD][8], const int (&rowu)[LD], const int (&offu)[LD], const int (&off8)[LD],
                                                 unsigned char* hi, unsigned char* lo, uint32_t chunk_bytes, float in_slope) {
#pragma unroll
  for (int u = 0; u < LD; u++) {
    if (rowu[u] < 0) continue;
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      float a0 = src[u][2 * j], a1 = src[u][2 * j + 1];
      if (LRELU) {
        a0 = fmaxf(a0, a0 * in_slope);                 // leaky_relu for 0 <= slope <= 1
        a1 = fmaxf(a1, a1 * in_slope);
      }
      hw[j] = cvt_f16x2_sat(a0, a1);
      const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[j]));
      if (F8) {
        const uint32_t l8 = cvt_e4m3x2_sat((a0 - hf.x) * TC_F8_LO_SCALE, (a1 - hf.y) * TC_F8_LO_SCALE);   // a - hi is exact in fp32
        const uint32_t h8 = cvt_e4m3x2_sat(hf.x, hf.y);                                                    // TC_F8_HI_SCALE == 1
        if (j & 1) { lw[j >> 1] |= l8 << 16; lw[2 + (j >> 1)] |= h8 << 16; }
        else { lw[j >> 1] = l8; lw[2 + (j >> 1)] = h8; }
      } else {
        lw[j] = cvt_f16x2_sat(a0 - hf.x, a1 - hf.y);
      }
    }
    *reinterpret_cast<uint4*>(hi + offu[u]) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    if (F8) {
      *reinterpret_cast<uint2*>(lo + off8[u]) = make_uint2(lw[0], lw[1]);                 // E4M3 lo of these 8 channels
      *reinterpret_cast<uint2*>(lo + off8[u] + chunk_bytes) = make_uint2(lw[2], lw[3]);   // E4M3 hi of these 8 channels
    } else {
      *reinterpret_cast<uint4*>(lo + offu[u]) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
    }
  }
}

// Epilogue of one consumer warpgroup: its 64 rows of the tile straight from the accumulator fragments (see wgmma.cuh): thread
// (warp w, lane l) owns rows 16w + l/4 and +8, column pairs 8j + 2(l%4).  The split-term accumulators are summed here in fp32
// round-to-nearest.  bias / res / row_lens may be NULL; acc_in: add alpha*value to y instead of overwriting it.  Rows >= tend (T, or n_b
// of a ragged batch) are not written.
template <int ACT, int NB, int TG>
__device__ __forceinline__ void tc_epilogue(const TcP& p, float (&acc)[TG][NB / 2], const Item& it, int row_base, int tend, const float* bias,
                                            const float* res, const int* row_lens, int acc_in, float inv_ws) {
  const int lane = threadIdx.x & 31;
  const int n0 = it.nblk * NB + 2 * (lane & 3);
  const int len_b = row_lens ? min(row_lens[it.b], p.T) : p.T;
  const float slope = p.out_slope, alpha = p.alpha;
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int t = row_base + (lane >> 2) + 8 * h;
    if (t >= tend) continue;
    const bool live = t < len_b;
    float* yrow = p.y + (long long)it.b * p.ybs + (long long)t * p.yrs + n0;
    const float* rrow = res ? res + (long long)it.b * p.rbs + (long long)t * p.rrs + n0 : nullptr;
#pragma unroll
    for (int j = 0; j < NB / 8; j++) {
      float a0 = acc[0][4 * j + 2 * h], a1 = acc[0][4 * j + 2 * h + 1];
      if (TG == 2) { a0 += acc[TG - 1][4 * j + 2 * h]; a1 += acc[TG - 1][4 * j + 2 * h + 1]; }
      float2 bv = make_float2(0.f, 0.f);
      if (bias) bv = __ldg(reinterpret_cast<const float2*>(bias + n0 + 8 * j));
      float2 o;
      o.x = tc_act<ACT>(fmaf(a0, inv_ws, bv.x), slope);    // inv_ws is a power of two: exact
      o.y = tc_act<ACT>(fmaf(a1, inv_ws, bv.y), slope);
      if (rrow) {
        const float2 rv = *reinterpret_cast<const float2*>(rrow + 8 * j);
        o.x += rv.x; o.y += rv.y;
      }
      if (acc_in) {
        const float2 yv = *reinterpret_cast<const float2*>(yrow + 8 * j);
        o.x = o.x * alpha + yv.x; o.y = o.y * alpha + yv.y;
      } else {
        o.x *= alpha; o.y *= alpha;
      }
      if (!live) o = make_float2(0.f, 0.f);
      *reinterpret_cast<float2*>(yrow + 8 * j) = o;
    }
  }
}

// Releases a slab / weight stage once every consumer warp has seen its MMAs retire (one arrival per consumer warp).
__device__ __forceinline__ void tc_release(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// RAG: ragged batch (TcP::x_lens != NULL).  A template parameter rather than a runtime branch: the cursor state would otherwise raise the
// padded path's spills (every NB is at the 96-register cap of one 544-thread CTA per SM).
template <int NB, bool RAG>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const TcP p) {
  constexpr int TG = NB <= 64 ? 2 : 1;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int R = p.R, SA = p.SA, SB = p.SB;
  const uint32_t a_plane = (uint32_t)TC_CHUNKS * R * 16;          // bytes of one hi (or lo) slab
  const uint32_t b_plane = (uint32_t)TC_CHUNKS * NB * 16;         // bytes of one hi (or lo) weight tile
  unsigned char* a_base = smem_raw;                                // [SA][hi|lo][chunk][R][16 B]
  unsigned char* b_base = a_base + (size_t)SA * 2 * a_plane;       // [SB][hi|lo][chunk][NB][16 B]
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_base + (size_t)SB * p.TPS * 2 * b_plane);
  uint64_t* fullA = bars;                  // [SA_MAX]
  uint64_t* emptyA = fullA + TC_SA_MAX;    // [SA_MAX]
  uint64_t* fullB = emptyA + TC_SA_MAX;    // [SB_MAX]
  uint64_t* emptyB = fullB + TC_SB_MAX;    // [SB_MAX]

  const int KBLOCKS = p.Cin / TC_KB;
  constexpr int CWARPS = TC_CTHREADS / 32;
  // Ragged batch: every role walks the compacted item sequence (RaggedWalk) in the same order, which keeps the rings' stage / phase
  // sequence identical across the three roles.
  constexpr bool rag = RAG;
  RaggedWalk walk{};
  int n_items = p.n_items;
  if (rag) { walk.init(p.x_lens, p.lens_scale, p.T, p.B, 128); n_items = walk.live * (p.N / p.NB); }

  if (tid == 0) {
    for (int i = 0; i < TC_SA_MAX; i++) { mbar_init(&fullA[i], TC_TW); mbar_init(&emptyA[i], CWARPS); }
    for (int i = 0; i < TC_SB_MAX; i++) { mbar_init(&fullB[i], 1); mbar_init(&emptyB[i], CWARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == CWARPS) {
    // ===================== weight-stage producer (TMA bulk copies) =====================
    if (lane == 0) {
      const uint32_t stage_bytes = 2 * b_plane;   // one tap of one K-block (hi + lo)
      Ring rb;
      const int per_blk = rag ? max(walk.live, 1) : p.B * p.tiles_per_batch;
      int nblk = (int)blockIdx.x / per_blk, rem = (int)blockIdx.x - nblk * per_blk;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        for (int seg = 0; seg < p.nseg; seg++) {
          const unsigned char* src = reinterpret_cast<const unsigned char*>(p.wt) + (long long)seg * p.seg_wbytes + TC_HDR +
                                     (size_t)nblk * p.taps * KBLOCKS * stage_bytes;   // tiles are ordered [kb][tap]
          for (int kb = 0; kb < KBLOCKS; kb++) {
            for (int tap = 0; tap < p.taps; tap += p.TPS) {
              const int n = min(p.TPS, p.taps - tap);
              const uint32_t bytes = (uint32_t)n * stage_bytes;
              mbar_wait(&emptyB[rb.idx], rb.phase ^ 1);
              mbar_expect_tx(&fullB[rb.idx], bytes);
              bulk_g2s(b_base + (size_t)rb.idx * p.TPS * stage_bytes, src, bytes, &fullB[rb.idx]);
              src += bytes;
              rb.advance(SB);
            }
          }
        }
        rem += (int)gridDim.x;
        while (rem >= per_blk) { rem -= per_blk; nblk++; }
      }
    }
  } else if (warp < CWARPS) {
    // ===================== consumer warpgroups: MMAs + epilogue =====================
    // Every operand is a precomputed descriptor base plus a constant.  A stage is released one MMA group late (wgmma.wait_group 1),
    // so the tensor core always has the next stage's MMAs queued while the previous ones retire.
    const int g = warp >> 2;                             // 64-row half of the tile
    const uint64_t a_const = wgmma_desc(0, (uint32_t)R * 16, 128), b_const = wgmma_desc(0, (uint32_t)NB * 16, 128);
    const float inv_ws0 = __ldg(p.wt);                 // header: 1 / (power-of-two weight scale)
    Ring ra, rb;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
      const Item it = rag ? walk.item(p.x_lens, p.lens_scale, p.T, 128, item) : decode_item(p, item);
      const int tend = rag ? walk.rows : p.T;
      for (int seg = 0; seg < p.nseg; seg++) {
        float acc[TG][NB / 2];
#pragma unroll
        for (int gg = 0; gg < TG; gg++)
#pragma unroll
          for (int i = 0; i < NB / 2; i++) acc[gg][i] = 0.f;
        int pend_b = -1, pend_a = -1;                  // stages whose MMAs are in the last committed group
        for (int kb = 0; kb < KBLOCKS; kb++, ra.advance(SA)) {
          const uint32_t sa = ra.idx;
          mbar_wait(&fullA[sa], ra.phase);
          const uint64_t a_hi = a_const | (uint64_t)((smem_u32(a_base + (size_t)sa * 2 * a_plane) >> 4) + 64 * g);
          const uint64_t a_lo = a_hi + (a_plane >> 4);
          uint32_t row_off = 0;
          for (int tap = 0; tap < p.taps; tap += p.TPS, rb.advance(SB)) {
            const uint32_t sb = rb.idx;
            const int n = min(p.TPS, p.taps - tap);
            mbar_wait(&fullB[sb], rb.phase);
            wgmma_fence();
            uint64_t b_hi = b_const | (uint64_t)(smem_u32(b_base + (size_t)sb * p.TPS * 2 * b_plane) >> 4);
            for (int j = 0; j < n; j++, b_hi += (2 * b_plane) >> 4, row_off += (uint32_t)p.dil) {
              const uint64_t b_lo = b_hi + (b_plane >> 4);
              const uint64_t ah0 = a_hi + row_off, al0 = a_lo + row_off;
              const uint32_t first = (kb | tap | j) ? 1u : 0u;
              if (TG == 2 && p.f8) {                         // (the host plans f8 work items with NB <= 64, i.e. TG == 2)
                Wgmma<NB>::f16(acc[0], ah0, b_hi, first);                        // fp16: A_hi * B_hi
                Wgmma<NB>::e4m3(acc[TG - 1], al0, b_lo, first);                  // E4M3, K = 32: [A_lo | A_hi] * [B_hi ; B_lo]
              } else {
                Wgmma<NB>::f16(acc[TG - 1], al0, b_hi, first);                   // A_lo * B_hi
                Wgmma<NB>::f16(acc[0], ah0, b_hi, TG >= 2 ? first : 1u);         // A_hi * B_hi
                Wgmma<NB>::f16(acc[TG - 1], ah0, b_lo, 1u);                      // A_hi * B_lo
              }
            }
            wgmma_commit();
            wgmma_wait<1>();                           // the previous group has retired: its stages may be refilled
            if (pend_b >= 0) tc_release(&emptyB[pend_b]);
            if (pend_a >= 0) { tc_release(&emptyA[pend_a]); pend_a = -1; }
            pend_b = (int)sb;
          }
          pend_a = (int)sa;
        }
        wgmma_wait<0>();
#pragma unroll
        for (int gg = 0; gg < TG; gg++) wgmma_keep<NB>(acc[gg]);
        if (pend_b >= 0) tc_release(&emptyB[pend_b]);
        if (pend_a >= 0) tc_release(&emptyA[pend_a]);
        // K-segmented conv: unit (item, seg) adds slice seg of the tile into y -- bias with the first slice; residual, alpha-free sum
        // and the pad-row mask with the last.  The same thread owns the same outputs in every unit, so the fp32 read-modify-write of
        // y needs no further ordering.  No output activation (checked on the host).
        const bool first = seg == 0, last = seg == p.nseg - 1;
        const float* bias = first ? p.bias : nullptr;
        const float* res = last ? p.res : nullptr;
        const int* lens = last ? p.row_lens : nullptr;
        const int acc_in = (!first || p.accumulate) ? 1 : 0;
        const float inv_ws = p.nseg == 1 ? inv_ws0
            : __ldg(reinterpret_cast<const float*>(reinterpret_cast<const unsigned char*>(p.wt) + (long long)seg * p.seg_wbytes));
        const int row_base = it.t0 + 64 * g + 16 * (warp & 3);
        switch (p.out_act) {                           // uniform branch: keeps tanhf out of the other variants' inner loops
          case FS2_ACT_RELU: tc_epilogue<FS2_ACT_RELU, NB, TG>(p, acc, it, row_base, tend, bias, res, lens, acc_in, inv_ws); break;
          case FS2_ACT_TANH: tc_epilogue<FS2_ACT_TANH, NB, TG>(p, acc, it, row_base, tend, bias, res, lens, acc_in, inv_ws); break;
          case FS2_ACT_LRELU: tc_epilogue<FS2_ACT_LRELU, NB, TG>(p, acc, it, row_base, tend, bias, res, lens, acc_in, inv_ws); break;
          default: tc_epilogue<FS2_ACT_NONE, NB, TG>(p, acc, it, row_base, tend, bias, res, lens, acc_in, inv_ws); break;
        }
      }
    }
  } else {
    // ===================== transform warps (activation + fp16 hi/lo split) =====================
    // The instruction count per (row, K-chunk) unit sets the speed of the narrow / small-k layers, so: one 32-byte sector per unit,
    // addresses from a per-K-block base + a precomputed 32-bit offset, no range checks for interior work items, the fp16 clamp
    // folded into the saturating convert, the input activation resolved outside the unit loop.
    const int wt = tid - (TC_CTHREADS + 32);           // 0..TC_TTHREADS-1
    const int rows_needed = 128 + (p.taps - 1) * p.dil;
    const int items = rows_needed * TC_CHUNKS;
    // Register ring of TC_DEPTH K-blocks: the loads of K-block seq + TC_DEPTH (possibly of a later work item) are issued as
    // soon as K-block seq has been converted and stored.
    constexpr int LD = TC_LD;                          // (row, chunk) units per thread per K-block
    constexpr int DEPTH = TC_DEPTH;                    // K-blocks in flight (register ring)
    float v[DEPTH][LD][8];
    const bool lrelu_in = p.in_act == FS2_ACT_LRELU;
    const float in_slope = p.in_slope;
    // per-thread (row, chunk) slots: fixed for the whole kernel
    int rowu[LD], offu[LD], off8[LD], goff[LD];
#pragma unroll
    for (int u = 0; u < LD; u++) {
      const int idx = u * TC_TTHREADS + wt;
      rowu[u] = idx < items ? (idx >> 1) : -1;
      offu[u] = (((idx & 1) * R) + (idx >> 1)) * 16;                  // smem byte offset inside a hi / lo plane
      off8[u] = (idx >> 1) * 16 + (idx & 1) * 8;                      // f8 split: byte offset inside one 16-channel E4M3 chunk
      goff[u] = (idx >> 1) * (int)p.xrs + (idx & 1) * 8;              // global float offset from the slab's first row
    }
    // load cursor (runs TC_DEPTH K-blocks ahead of the store cursor); no divisions on the per-K-block path
    int l_item = blockIdx.x, l_kb = 0, l_seg = 0;
    const float* l_xrow = nullptr;                     // &x[b][t0 - pad][0]; rows outside [0, l_tend) are never dereferenced
    int l_tfirst = 0, l_tend = p.T;                    // l_tend: T, or n_b of a ragged batch
    bool l_interior = false;                           // warp-uniform: every slab row of the item exists
    auto l_set_item = [&]() {
      if (l_item < n_items) {
        const Item it = rag ? walk.item(p.x_lens, p.lens_scale, p.T, 128, l_item) : decode_item(p, l_item);
        if (rag) l_tend = walk.rows;
        const int s_tap = l_seg / p.seg_nkc, s_kc = l_seg - s_tap * p.seg_nkc;   // K-segment: one tap, one 256-channel chunk (0, 0 when nseg == 1)
        l_tfirst = it.t0 - p.pad + s_tap;
        l_xrow = p.x + (long long)it.b * p.xbs + (long long)l_tfirst * p.xrs + s_kc * p.Cin;
        l_interior = l_tfirst >= 0 && l_tfirst + rows_needed <= l_tend;
      }
    };
    l_set_item();
    auto issue_loads = [&](float (&dst)[LD][8]) {     // loads K-block (l_item, l_kb), then advances the load cursor
      const float* xk = l_xrow + l_kb * TC_KB;
      if (l_interior) {
#pragma unroll
        for (int u = 0; u < LD; u++)
          if (rowu[u] >= 0) ldg256(dst[u], xk + goff[u]);
      } else {
#pragma unroll
        for (int u = 0; u < LD; u++) {
          const int t = l_tfirst + rowu[u];
          if (rowu[u] >= 0 && t >= 0 && t < l_tend) {
            ldg256(dst[u], xk + goff[u]);
          } else {
#pragma unroll
            for (int j = 0; j < 8; j++) dst[u][j] = 0.f;              // conv zero padding
          }
        }
      }
      if (++l_kb == KBLOCKS) {
        l_kb = 0;
        if (++l_seg == p.nseg) { l_seg = 0; l_item += gridDim.x; }
        l_set_item();
      }
    };
    const int my_items = (n_items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // >= 0: blockIdx.x < gridDim.x
    const int total = my_items * p.nseg * KBLOCKS;
#pragma unroll
    for (int d = 0; d < DEPTH; d++)
      if (d < total) issue_loads(v[d]);
    Ring ra;
    for (int base = 0; base < total; base += DEPTH) {
#pragma unroll
      for (int d = 0; d < DEPTH; d++) {
        const int seq = base + d;
        if (seq < total) {
          mbar_wait(&emptyA[ra.idx], ra.phase ^ 1);
          unsigned char* hi = a_base + (size_t)ra.idx * 2 * a_plane;
          if (p.f8) {
            if (lrelu_in) tc_convert_store<true, true, LD>(v[d], rowu, offu, off8, hi, hi + a_plane, (uint32_t)R * 16, in_slope);
            else tc_convert_store<false, true, LD>(v[d], rowu, offu, off8, hi, hi + a_plane, (uint32_t)R * 16, in_slope);
          } else {
            if (lrelu_in) tc_convert_store<true, false, LD>(v[d], rowu, offu, off8, hi, hi + a_plane, (uint32_t)R * 16, in_slope);
            else tc_convert_store<false, false, LD>(v[d], rowu, offu, off8, hi, hi + a_plane, (uint32_t)R * 16, in_slope);
          }
          fence_proxy_async();                         // generic-proxy stores -> visible to the tensor core (async proxy)
          __syncwarp();
          if (lane == 0) mbar_arrive(&fullA[ra.idx]);   // one arrival per transform warp
          ra.advance(SA);
          if (seq + DEPTH < total) issue_loads(v[d]);
        }
      }
    }
  }
}

// The NB instantiations live in their own translation units (conv_tc_nb*.cu) so that the library builds in parallel.
// conv_tc_prepare_nb / conv_tc_launch_nb return cudaErrorInvalidValue for an NB they do not instantiate.
#define FS2_CONV_TC_NB_DECL(nb)                        \
  cudaError_t conv_tc_prepare_nb##nb(int smem_bytes); \
  void conv_tc_launch_nb##nb(const TcP& p, unsigned grid, size_t smem, cudaStream_t s);
FS2_CONV_TC_NB_DECL(16) FS2_CONV_TC_NB_DECL(32) FS2_CONV_TC_NB_DECL(48) FS2_CONV_TC_NB_DECL(64)
FS2_CONV_TC_NB_DECL(80) FS2_CONV_TC_NB_DECL(96) FS2_CONV_TC_NB_DECL(112) FS2_CONV_TC_NB_DECL(128)
#undef FS2_CONV_TC_NB_DECL

#define FS2_CONV_TC_NB_DEF(nb)                                                                          \
  cudaError_t conv_tc_prepare_nb##nb(int smem_bytes) {                                                  \
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<nb, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes); \
    return e == cudaSuccess ? cudaFuncSetAttribute(conv_tc_kernel<nb, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes) : e; \
  }                                                                                                     \
  void conv_tc_launch_nb##nb(const TcP& p, unsigned grid, size_t smem, cudaStream_t s) {                \
    if (p.x_lens) conv_tc_kernel<nb, true><<<grid, TC_THREADS, smem, s>>>(p);                          \
    else conv_tc_kernel<nb, false><<<grid, TC_THREADS, smem, s>>>(p);                                  \
  }

}  // namespace fs2
