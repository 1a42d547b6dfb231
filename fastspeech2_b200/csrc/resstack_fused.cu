// One persistent wgmma kernel per HiFi-GAN upsample stage for the multi-receptive-field ResBlock group
//
//   y = (1/n_kernels) * sum_j ResBlock_j(x),   ResBlock_j: x <- conv_{k_j,1}(lrelu(conv_{k_j,d}(lrelu(x)))) + x  for d in dilations
//
// (hifigan/models.py:154-160 and ResBlock.forward :96-103; contract: fs2_resstack in include/fs2b200.h).  The per-layer design
// issues 18 conv launches per stage and moves every intermediate through HBM (~48 full-tensor passes); here a CTA owns one time
// tile of one utterance and keeps the whole chain on chip:
//
//   * slab = MT*128 rows starting H (the sum of the receptive radii) rows before the tile: every conv is evaluated on the full
//     slab, garbage from the slab edges grows inward by one conv radius per layer and by construction stays inside the H-row halo
//     (halo recompute); rows outside the utterance [0, N) are forced to zero after every layer (Conv1d zero padding).
//   * activations live in shared memory ALREADY in tensor-core operand form: per 16-channel K-block an fp16 "hi" plane and an
//     E4M3 plane [lo * 2^12 | hi] (the two-MMA operand split of conv_tc_kernel.cuh, FS2_TC_VARIANT_F8), no-swizzle K-major
//     [16-byte K-chunk][row][16 B], so a conv tap is the same slab with the descriptor start advanced by tap*dilation rows.
//     Two slabs: XA = lrelu(x) (conv1's operand), XT = lrelu(conv1 output) (conv2's operand).
//   * two consumer warpgroups own the 64-row blocks g*MT .. g*MT + MT-1 of the slab and keep their accumulators in registers: one
//     for the FP16 main term and one for the E4M3 correction (Hopper accumulates E4M3 products with reduced precision, so the
//     correction must not be added into the main term's accumulator).  The residual stream x (fp32) stays in shared memory in the
//     same fragment order (each thread reads back only what it wrote).  Epilogue = accumulators -> bias / residual / lrelu ->
//     operand split -> st.shared into the other slab; a named barrier over both warpgroups publishes it (the next conv's taps
//     read the neighbours' rows).
//   * weights stream through a cp.async.bulk ring exactly as in conv_tc_kernel.cuh (same tile images: the packer's f8 format).
//   * global I/O is TMA with tensor maps: the fp32 tile of x arrives as 3-D boxes [1][128 rows][32 channels] (128-byte swizzle;
//     rows outside [0, N) are zero-filled by the hardware = the conv's zero padding, and there is no bleed between utterances)
//     into XT while it is idle; the result leaves as boxes staged in XA with a TMA store (first kernel size) or TMA reduce-add
//     (the others: the mean over kernel sizes accumulates in L2).  HBM sees x once per kernel size and y once.
//
// Roles: warps 0-7 two consumer warpgroups (conversion, MMAs, epilogues; thread 0 issues the tensor-map copies), warp 8 weight producer.
#include <cuda.h>

#include "conv_tc_kernel.cuh"

namespace fs2 {

constexpr int RS_MAXK = FS2_MAX_DIL + 4;   // kernel sizes per stage
constexpr int RS_GUARD = 1024;             // zeroed bytes in front of the first slab (taps reach up to 32 rows before row 0)
constexpr int RS_SB_MAX = 16;
constexpr int RS_THREADS = 256 + 32;

struct RsConv { const unsigned char* w; const float* b; int taps, dil; };
struct RsP {
  int B, N;
  int n_kernels, n_dil;
  RsConv conv[RS_MAXK][FS2_MAX_DIL][2];
  int H, TILE, tiles_per_b, n_items;
  float alpha;
  int SB;
  int OBOX, n_oboxes;            // rows per output box (TILE = n_oboxes * OBOX, OBOX % 8 == 0)
  int TPS;                       // conv taps per weight stage (one bulk copy / one handshake)
  int accumulate;                // the first kernel size reduce-adds into y too
  const int* lens; int lens_scale;   // ragged batch (fs2_resstack_args::lens) or NULL; n_items then only bounds the grid
};

// ------------------------------------------------------------------ TMA (tensor-map) wrappers
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int c0, int n0, int b, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
                   smem_u32(dst)),
               "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(n0), "r"(b), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* tm, int c0, int n0, int b, const void* src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(reinterpret_cast<uint64_t>(tm)),
               "r"(c0), "r"(n0), "r"(b), "r"(smem_u32(src))
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* tm, int c0, int n0, int b, const void* src) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(
                   reinterpret_cast<uint64_t>(tm)),
               "r"(c0), "r"(n0), "r"(b), "r"(smem_u32(src))
               : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_reads() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }   // both consumer warpgroups
// byte offset of 16-byte chunk c of row r inside a [rows][128 B] box written / read by TMA with CU_TENSOR_MAP_SWIZZLE_128B
__device__ __forceinline__ uint32_t sw128(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

__device__ __forceinline__ float rs_lrelu(float v) { return fmaxf(v, 0.1f * v); }   // LRELU_SLOPE = 0.1 (hifigan/models.py:7)

// channels c, c+1 (c even) of slab row `row` -> the operand planes (fp16 hi; E4M3 [lo * 2^12 | hi]).  `a0`, `a1` already carry the
// activation and the out-of-utterance zeroing.
__device__ __forceinline__ void rs_store2(unsigned char* slab, uint32_t chunk_bytes, int row, int c, float a0, float a1) {
  const uint32_t hw = cvt_f16x2_sat(a0, a1);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw));
  const uint32_t l8 = cvt_e4m3x2_sat((a0 - hf.x) * TC_F8_LO_SCALE, (a1 - hf.y) * TC_F8_LO_SCALE);
  const uint32_t h8 = cvt_e4m3x2_sat(hf.x, hf.y);          // TC_F8_HI_SCALE == 1
  const int cc = c & 15;
  unsigned char* kblk = slab + (size_t)(c >> 4) * 4 * chunk_bytes + (size_t)row * 16;
  *reinterpret_cast<uint32_t*>(kblk + (cc >> 3) * chunk_bytes + (cc & 7) * 2) = hw;
  *reinterpret_cast<unsigned short*>(kblk + 2 * chunk_bytes + cc) = (unsigned short)l8;
  *reinterpret_cast<unsigned short*>(kblk + 3 * chunk_bytes + cc) = (unsigned short)h8;
}

// RAG: ragged batch (RsP::lens != NULL), a template parameter so that the padded path's code and register allocation stay as they are.
template <int C, int MT, bool RAG>
__global__ void __launch_bounds__(RS_THREADS, 1) resstack_kernel(const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmy,
                                                                 const RsP p) {
  constexpr int KB = C / 16, R = MT * 128, NH = C / 32, NJ = C / 8;   // NJ: 8-column fragment groups of a row
  constexpr uint32_t CHUNK = (uint32_t)R * 16, PLANE = 2 * CHUNK, KBLK = 2 * PLANE, SLAB = KB * KBLK;
  constexpr uint32_t WSTAGE = 64u * C;
  constexpr uint32_t XBOX = 128 * 128;                                 // bytes of one input box [128 rows][32 ch] fp32
  static_assert(SLAB == (uint32_t)R * C * 4, "an operand slab has exactly the size of the fp32 tile it is built from");
  static_assert(MT * (C / 2) * 256 * 4 == SLAB, "the residual stream has the size of a slab");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  unsigned char* smem0 = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // swizzle atoms are 1024 bytes
  unsigned char* xa = smem0 + RS_GUARD;          // 1024-byte aligned: doubles as the swizzled staging area of the result
  unsigned char* xt = xa + SLAB;                 //                    doubles as the landing area of the fp32 input boxes
  float* xres = reinterpret_cast<float*>(xt + SLAB);   // residual stream [MT][C/2 fragment registers][256 consumer threads]
  unsigned char* ring = xt + 2 * SLAB;
  const uint32_t stage_bytes = (uint32_t)p.TPS * WSTAGE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + (size_t)p.SB * stage_bytes);
  uint64_t* fullB = bars;                       // [RS_SB_MAX]
  uint64_t* emptyB = fullB + RS_SB_MAX;         // [RS_SB_MAX]
  uint64_t* xLoaded = emptyB + RS_SB_MAX;       // the round's input boxes have landed in XT

  for (int i = tid; i < RS_GUARD / 16; i += RS_THREADS) reinterpret_cast<uint4*>(smem0)[i] = make_uint4(0, 0, 0, 0);
  if (tid == 0) {
    for (int i = 0; i < RS_SB_MAX; i++) { mbar_init(&fullB[i], 1); mbar_init(&emptyB[i], 8); }
    mbar_init(xLoaded, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmx)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmy)) : "memory");
  }
  fence_proxy_async();
  __syncthreads();
  // ragged batch: the producer and both consumer warpgroups walk the same compacted item sequence (RaggedWalk, conv_tc_kernel.cuh)
  RaggedWalk walk{};
  int n_items = p.n_items;
  if (RAG) { walk.init(p.lens, p.lens_scale, p.N, p.B, p.TILE); n_items = walk.live; }

  if (warp == 8) {
    // ===================== weight producer: every conv's stages once per work item and kernel size =====================
    if (lane == 0) {
      Ring rb;
      for (int item = blockIdx.x; item < n_items; item += gridDim.x)
        for (int j = 0; j < p.n_kernels; j++)
          for (int d = 0; d < p.n_dil; d++)
            for (int c2 = 0; c2 < 2; c2++) {
              const RsConv cv = p.conv[j][d][c2];
              const unsigned char* src = cv.w + TC_HDR;   // tiles are ordered [kb][tap]: the taps of one K-block are contiguous
              for (int kb = 0; kb < KB; kb++)
                for (int tap = 0; tap < cv.taps; tap += p.TPS) {
                  const uint32_t bytes = (uint32_t)min(p.TPS, cv.taps - tap) * WSTAGE;
                  mbar_wait(&emptyB[rb.idx], rb.phase ^ 1);
                  mbar_expect_tx(&fullB[rb.idx], bytes);
                  bulk_g2s(ring + (size_t)rb.idx * stage_bytes, src, bytes, &fullB[rb.idx]);
                  src += bytes;
                  rb.advance((uint32_t)p.SB);
                }
            }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int g = warp >> 2, w = warp & 3;
  const bool io = tid == 0;                      // issues every tensor-map copy (bulk groups are per thread)
  const uint64_t a_const = wgmma_desc(0, CHUNK, 128), b_const = wgmma_desc(0, (uint32_t)C * 16, 128);
  const uint32_t xa16 = smem_u32(xa) >> 4, xt16 = smem_u32(xt) >> 4;
  const int rbase = 64 * MT * g + 16 * w + (lane >> 2);   // slab row of fragment (block i, half h): rbase + 64 i + 8 h
  const int cbase = 2 * (lane & 3);                       // channel of fragment column group jj: cbase + 8 jj
  float acc[MT][C / 2], corr[MT][C / 2];                  // FP16 main term | E4M3 correction
  auto xr = [&](int i, int r) -> float& { return xres[(i * (C / 2) + r) * 256 + tid]; };   // residual stream, fragment layout
  Ring rb;
  uint32_t round_phase = 0;
  bool stores_pending = false;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    int b, t0, nrows = p.N;                         // nrows: rows of utterance b (n_b of a ragged batch); the convs pad at its end
    if (RAG) {
      const Item it = walk.item(p.lens, p.lens_scale, p.N, p.TILE, item);
      b = it.b; t0 = it.t0; nrows = walk.rows;
    } else {
      b = item / p.tiles_per_b;
      t0 = (item - b * p.tiles_per_b) * p.TILE;
    }
    for (int j = 0; j < p.n_kernels; j++) {
      // ---- input: TMA boxes of x -> XT (idle: the last conv that read it has retired), then residual stream -> registers, lrelu(x) -> XA
      if (io) {
        if (stores_pending) tma_wait_reads();           // previous result boxes have been read out of XA
        mbar_expect_tx(xLoaded, (uint32_t)(MT * NH) * XBOX);
        for (int hh = 0; hh < NH; hh++)
          for (int m = 0; m < MT; m++) tma_load_3d(xt + (size_t)(hh * MT + m) * XBOX, &tmx, hh * 32, t0 - p.H + m * 128, b, xLoaded);
      }
      stores_pending = true;
      consumers_sync();                                 // XA is free
      mbar_wait(xLoaded, round_phase);
#pragma unroll
      for (int i = 0; i < MT; i++)
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int row = rbase + 64 * i + 8 * h, m = row >> 7, r128 = row & 127;
#pragma unroll
          for (int jj = 0; jj < NJ; jj++) {
            const int c = cbase + 8 * jj;
            float2 u = *reinterpret_cast<const float2*>(xt + (size_t)((c >> 5) * MT + m) * XBOX + sw128(r128, (c & 31) >> 2) + (c & 3) * 4);
            if (RAG && t0 - p.H + row >= nrows) u = make_float2(0.f, 0.f);   // the padding of a ragged batch reads as zero
            xr(i, 4 * jj + 2 * h) = u.x;
            xr(i, 4 * jj + 2 * h + 1) = u.y;
            rs_store2(xa, CHUNK, row, c, rs_lrelu(u.x), rs_lrelu(u.y));   // rows outside the utterance arrive as zeros (TMA fill)
          }
        }
      fence_proxy_async();
      consumers_sync();                                 // XA complete; every thread has read the boxes, so XT may be overwritten
      for (int d = 0; d < p.n_dil; d++) {
        const bool last = d == p.n_dil - 1;
        for (int c2 = 0; c2 < 2; c2++) {
          const RsConv cv = p.conv[j][d][c2];
          const uint32_t slab16 = c2 == 0 ? xa16 : xt16;
          const int pad = (cv.taps - 1) * cv.dil / 2;
          // ---- MMAs: every tap of every K-block for this warpgroup's MT 64-row blocks; a weight stage is released one group late
          int pend = -1;
          for (int kb = 0; kb < KB; kb++) {
            const uint64_t a_hi = a_const | (uint64_t)((slab16 + kb * (KBLK >> 4) + 64 * MT * g) & 0x3fff);
            int row_off = -pad;
            for (int tap = 0; tap < cv.taps; tap += p.TPS, rb.advance((uint32_t)p.SB)) {
              const int n = min(p.TPS, cv.taps - tap);
              mbar_wait(&fullB[rb.idx], rb.phase);
              wgmma_fence();
              uint64_t b_hi = b_const | (uint64_t)(smem_u32(ring + (size_t)rb.idx * stage_bytes) >> 4);
              for (int t = 0; t < n; t++, b_hi += WSTAGE >> 4, row_off += cv.dil) {
                const uint64_t b_x8 = b_hi + ((2u * C * 16u) >> 4);
                const uint64_t ah0 = a_hi + (uint64_t)(int64_t)row_off;      // start-address field += rows (16 B each); never carries out of the field
                const uint64_t ax0 = ah0 + (PLANE >> 4);
                const uint32_t first = (kb | tap | t) ? 1u : 0u;
#pragma unroll
                for (int i = 0; i < MT; i++) Wgmma<C>::f16(acc[i], ah0 + i * 64, b_hi, first);
#pragma unroll
                for (int i = 0; i < MT; i++) Wgmma<C>::e4m3(corr[i], ax0 + i * 64, b_x8, first);
              }
              wgmma_commit();
              wgmma_wait<1>();
              if (pend >= 0) tc_release(&emptyB[pend]);
              pend = (int)rb.idx;
            }
          }
          wgmma_wait<0>();
#pragma unroll
          for (int i = 0; i < MT; i++) { wgmma_keep<C>(acc[i]); wgmma_keep<C>(corr[i]); }
          tc_release(&emptyB[pend]);
          // ---- epilogue straight from the fragments
          const float inv_s = __ldg(reinterpret_cast<const float*>(cv.w));
#pragma unroll
          for (int jj = 0; jj < NJ; jj++) {
            const int c = cbase + 8 * jj;
            const float2 bv = __ldg(reinterpret_cast<const float2*>(cv.b + c));
#pragma unroll
            for (int i = 0; i < MT; i++)
#pragma unroll
              for (int h = 0; h < 2; h++) {
                const int row = rbase + 64 * i + 8 * h;
                const int gr = t0 - p.H + row;
                const bool in = gr >= 0 && gr < nrows;
                const float s0 = acc[i][4 * jj + 2 * h] + corr[i][4 * jj + 2 * h], s1 = acc[i][4 * jj + 2 * h + 1] + corr[i][4 * jj + 2 * h + 1];
                float v0 = fmaf(s0, inv_s, bv.x), v1 = fmaf(s1, inv_s, bv.y);
                if (c2 == 0) {
                  // conv1: lrelu -> conv2's operand slab
                  rs_store2(xt, CHUNK, row, c, in ? rs_lrelu(v0) : 0.f, in ? rs_lrelu(v1) : 0.f);
                } else {
                  v0 += xr(i, 4 * jj + 2 * h); v1 += xr(i, 4 * jj + 2 * h + 1);   // + residual
                  if (!last) {
                    xr(i, 4 * jj + 2 * h) = v0; xr(i, 4 * jj + 2 * h + 1) = v1;
                    rs_store2(xa, CHUNK, row, c, in ? rs_lrelu(v0) : 0.f, in ? rs_lrelu(v1) : 0.f);
                  } else if (row >= p.H && row < p.H + p.TILE) {
                    // result of this kernel size, alpha * x (mean over kernel sizes, models.py:154-160), staged in XA (idle since conv1
                    // of this pair has retired) as swizzled [OBOX rows][32 channels] boxes for the TMA store / reduce-add
                    const int ro = row - p.H, bx = ro / p.OBOX, rb_ = ro - bx * p.OBOX;
                    unsigned char* obox = xa + (size_t)((c >> 5) * p.n_oboxes + bx) * ((size_t)p.OBOX * 128);
                    *reinterpret_cast<float2*>(obox + sw128(rb_, (c & 31) >> 2) + (c & 3) * 4) = make_float2(v0 * p.alpha, v1 * p.alpha);
                  }
                }
              }
          }
          fence_proxy_async();
          consumers_sync();                             // the next conv's taps read rows of both warpgroups
        }
      }
      round_phase ^= 1;
      // ---- result boxes -> y: store for the first kernel size, reduce-add (in L2) for the others; rows beyond N are clipped by the TMA
      if (io) {
        tma_wait_all();   // the previous kernel size's boxes are complete in L2 before this one's reduce-add
        for (int hh = 0; hh < NH; hh++)
          for (int bx = 0; bx < p.n_oboxes; bx++) {
            const unsigned char* src = xa + (size_t)(hh * p.n_oboxes + bx) * ((size_t)p.OBOX * 128);
            if (j == 0 && !p.accumulate) tma_store_3d(&tmy, hh * 32, t0 + bx * p.OBOX, b, src);
            else tma_reduce_add_3d(&tmy, hh * 32, t0 + bx * p.OBOX, b, src);
          }
        tma_commit();
      }
    }
  }
  if (io) tma_wait_all();
}

// ------------------------------------------------------------------ host side
static size_t rs_smem_bytes(int C, int MT, int SB, int TPS) {
  const size_t slab = (size_t)(C / 16) * 4 * (MT * 128) * 16;
  return RS_GUARD + 3 * slab + (size_t)SB * TPS * 64 * C + (2 * RS_SB_MAX + 2) * 8 + 16 + 1024;   // + worst-case 1024-byte alignment slack
}

// Launch plan (pure host logic): out[12] = {MT, H (halo rows per side), TILE (output rows per work item), work items, grid, weight ring
// stages, dynamic shared memory bytes, accumulator registers per consumer thread, rows per output box, output boxes per tile and
// 32-channel block, taps per weight stage, independent-tile mode (0: every work item is one slab with a halo at its two ends)}
int resstack_plan(const fs2_resstack_args* a, int num_sms, int* out) {
  if (!a || a->B <= 0 || a->N <= 0 || num_sms <= 0) return FS2_ERR_ARG;
  if (a->C != 32 && a->C != 64) return FS2_ERR_UNSUPPORTED;
  if (a->n_kernels <= 0 || a->n_kernels > RS_MAXK || a->n_dil <= 0 || a->n_dil > FS2_MAX_DIL) return FS2_ERR_ARG;
  int H = 0;
  for (int j = 0; j < a->n_kernels; j++) {
    const int k = a->k[j];
    if (k <= 0 || !(k & 1)) return FS2_ERR_UNSUPPORTED;
    int hj = 0;
    for (int d = 0; d < a->n_dil; d++) {
      const int dil = a->dil[j][d];
      if (dil <= 0 || (k - 1) * dil / 2 > 32) return FS2_ERR_UNSUPPORTED;      // taps reach at most 32 rows outside a tile (guard / neighbour tile)
      hj += (k - 1) * dil / 2 + (k - 1) / 2;
    }
    H = hj > H ? hj : H;
  }
  H = (H + 3) & ~3;                             // output boxes are whole swizzle atoms (multiples of 8 rows)
  // 128-row tiles per slab: the two warpgroups hold MT 64-row blocks each of fp32 main and correction accumulators (MT * C registers)
  const int MT = a->C == 32 ? 4 : 2;
  int TILE = 0, obox = 0, n_oboxes = 0;
  // the result leaves as TMA boxes of `obox` rows (a multiple of 8, <= 256) that tile TILE exactly: widen the halo by up to 32 rows
  // until TILE splits into at most 12 boxes (e.g. 384 - 2*4 = 376 = 47 x 8 would need 47 stores; 384 - 2*8 = 368 = 2 x 184)
  for (int hc = H; hc <= H + 32 && !obox; hc += 4) {
    const int tile = MT * 128 - 2 * hc;
    if (tile < 64) break;
    for (int r = 256; r >= 8; r -= 8)
      if (tile % r == 0 && tile / r <= 12) { TILE = tile; obox = r; H = hc; break; }
  }
  if (!obox) return FS2_ERR_UNSUPPORTED;
  n_oboxes = TILE / obox;
  const long long tiles_per_b = (a->N + TILE - 1) / TILE, items = tiles_per_b * a->B;
  if (items > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
  const int TPS = a->C == 32 ? 4 : 2;           // taps per weight stage: 8 KB stages (fewer handshakes per MMA; conv_tc measured -10..-25 %)
  int SB = 8;
  while (SB > 2 && rs_smem_bytes(a->C, MT, SB, TPS) > 227 * 1024) SB--;
  if (rs_smem_bytes(a->C, MT, SB, TPS) > 227 * 1024) return FS2_ERR_UNSUPPORTED;
  out[0] = MT; out[1] = H; out[2] = TILE; out[3] = (int)items; out[4] = items < num_sms ? (int)items : num_sms; out[5] = SB;
  out[6] = (int)rs_smem_bytes(a->C, MT, SB, TPS); out[7] = MT * a->C; out[8] = obox; out[9] = n_oboxes;
  out[10] = TPS; out[11] = 0;
  return FS2_OK;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
  static std::atomic<void*> cached{nullptr};
  void* f = cached.load(std::memory_order_acquire);
  if (!f) {
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess) return nullptr;
    cached.store(f, std::memory_order_release);
  }
  return reinterpret_cast<EncodeTiledFn>(f);
}
// fp32 [B][N][C] contiguous as a rank-3 map, boxes of [1][rows][32 channels] with the 128-byte swizzle, zero fill outside the tensor
static int make_map(CUtensorMap* tm, const float* base, int B, int N, int C, int box_rows) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return FS2_ERR_UNSUPPORTED;
  const cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)N, (cuuint64_t)B};
  const cuuint64_t strides[2] = {(cuuint64_t)C * 4, (cuuint64_t)N * C * 4};
  const cuuint32_t box[3] = {32, (cuuint32_t)box_rows, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? FS2_OK : FS2_ERR_CUDA - 1;
}

int resstack(const fs2_resstack_args* a, cudaStream_t s) {
  if (!a || !a->x || !a->y) return FS2_ERR_ARG;
  if (!aligned16(a->x) || !aligned16(a->y)) return FS2_ERR_ARG;
  if (a->B <= 0 || a->N <= 0 || a->C <= 0) return FS2_ERR_ARG;
  if (a->lens && a->lens_scale < 1) return FS2_ERR_ARG;
  {  // not in place: a work item re-reads halo rows of x that its neighbours' results would already have overwritten
    const unsigned char *xb = reinterpret_cast<const unsigned char*>(a->x), *yb = reinterpret_cast<const unsigned char*>(a->y);
    const size_t bytes = (size_t)a->B * a->N * a->C * sizeof(float);
    if (xb < yb + bytes && yb < xb + bytes) return FS2_ERR_ARG;
  }
  int derr = FS2_OK;
  DevState* dv = dev_state(&derr);
  if (!dv) return derr;
  int plan[12];
  FS2_TRY(resstack_plan(a, dv->num_sms.load(std::memory_order_relaxed), plan));
  if (!dv->fused_ready.load(std::memory_order_acquire)) {
    DevOnce once;
    if (!dv->fused_ready.load(std::memory_order_relaxed)) {
      const int mx = 227 * 1024;
      cudaError_t e = cudaFuncSetAttribute(resstack_kernel<32, 4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
      if (e == cudaSuccess) e = cudaFuncSetAttribute(resstack_kernel<64, 2, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
      if (e == cudaSuccess) e = cudaFuncSetAttribute(resstack_kernel<32, 4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
      if (e == cudaSuccess) e = cudaFuncSetAttribute(resstack_kernel<64, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, mx);
      if (e != cudaSuccess) return FS2_ERR_CUDA - (int)e;
      dv->fused_ready.store(true, std::memory_order_release);
    }
  }
  RsP p{};
  p.B = a->B; p.N = a->N;
  p.n_kernels = a->n_kernels; p.n_dil = a->n_dil;
  double flops = 0;
  for (int j = 0; j < a->n_kernels; j++)
    for (int d = 0; d < a->n_dil; d++) {
      if (!a->w1_tc[j][d] || !a->w2_tc[j][d] || !a->b1[j][d] || !a->b2[j][d]) return FS2_ERR_ARG;
      if (!aligned16(a->w1_tc[j][d]) || !aligned16(a->w2_tc[j][d]) || !aligned16(a->b1[j][d]) || !aligned16(a->b2[j][d])) return FS2_ERR_ARG;
      p.conv[j][d][0] = RsConv{reinterpret_cast<const unsigned char*>(a->w1_tc[j][d]), a->b1[j][d], a->k[j], a->dil[j][d]};
      p.conv[j][d][1] = RsConv{reinterpret_cast<const unsigned char*>(a->w2_tc[j][d]), a->b2[j][d], a->k[j], 1};
      flops += 2.0 * 2.0 * a->B * (double)a->N * a->C * a->C * a->k[j];
    }
  p.H = plan[1]; p.TILE = plan[2]; p.tiles_per_b = (a->N + p.TILE - 1) / p.TILE; p.n_items = plan[3];
  p.alpha = a->alpha > 0.f ? a->alpha : 1.f / (float)a->n_kernels; p.accumulate = a->accumulate; p.SB = plan[5]; p.OBOX = plan[8]; p.n_oboxes = plan[9]; p.TPS = plan[10];
  p.lens = a->lens; p.lens_scale = a->lens_scale;   // the grid stays the padded plan's: the host never reads device lengths
  alignas(64) CUtensorMap tmx, tmy;
  FS2_TRY(make_map(&tmx, a->x, a->B, a->N, a->C, 128));
  FS2_TRY(make_map(&tmy, a->y, a->B, a->N, a->C, p.OBOX));
  prof_before(s);
  if (a->C == 32) {
    if (a->lens) resstack_kernel<32, 4, true><<<plan[4], RS_THREADS, plan[6], s>>>(tmx, tmy, p);
    else resstack_kernel<32, 4, false><<<plan[4], RS_THREADS, plan[6], s>>>(tmx, tmy, p);
  } else {
    if (a->lens) resstack_kernel<64, 2, true><<<plan[4], RS_THREADS, plan[6], s>>>(tmx, tmy, p);
    else resstack_kernel<64, 2, false><<<plan[4], RS_THREADS, plan[6], s>>>(tmx, tmy, p);
  }
  prof_after(s, 0, flops);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
