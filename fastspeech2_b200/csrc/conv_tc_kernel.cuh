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
// Persistent, warp-specialised kernel: one CTA per SM walks a list of work items (one 128-row time tile of one utterance x NG
// blocks of NB <= 128 output channels); four roles overlap through mbarrier rings:
//   warp 8      weight producer: every (tap, 16-channel K-block) weight stage is ONE cp.async.bulk (TMA bulk engine) of a
//               host-pre-split, host-pre-tiled smem image  [hi|lo][16-byte K-chunk][n][8 halfs].
//   warps 9-16  activation transform: read the [128 + (taps-1)*dil] x 16-channel slab of a K-block ONCE from global
//               (one 32-byte sector per row and 8 channels, a register ring of K-blocks in flight), apply the input activation,
//               split hi/lo and store both in the no-swizzle K-major layout [16-byte K-chunk][row][8 halfs].  There a core
//               matrix (8 rows x 16 B) starting at ANY row is 128 contiguous bytes, so each conv tap is just the same slab with
//               the descriptor start address advanced by tap*dil rows: the slab is loaded and split once per K-block, not once per tap.
//               With NG > 1 the item's Cin/16 K-block slabs stay resident (SA >= Cin/16, one plan field) while the consumers run
//               the K loop once per channel block, so the slab is loaded and split once per tile rather than once per block, and
//               the tile's input is read from global once; each stage is released on the item's last block (ring_release_last).
//   warps 0-7   two consumer warpgroups, 64 output rows each: per weight stage 3 (split terms) wgmma m64nNBk16 with register
//               accumulators (or one FP16 + one E4M3 K = 32 MMA, TcP::f8), then the epilogue straight from the accumulator
//               fragments: bias / activation / residual / alpha / accumulate / pad-row mask -> global stores.  The residual and
//               the y to accumulate into come from shared memory (below), so the epilogue reads only registers and shared memory.
//   warp 17     staging (only for a conv with a residual, accumulate or K-segments): per work item and consumer warp, one
//               cp.async.bulk per row of the residual and of the old y into that warp's 16 rows of a shared tile (TcStage), while
//               the item's MMAs run.  Read from global in the epilogue, each of those loads sat behind the previous y store (y may
//               alias both, so ptxas keeps them in order): one serial DRAM round trip per 8 columns with no MMA issuing.  A
//               K-segmented conv keeps its running fp32 slice sum in the same tile instead of reading y back per slice.
#pragma once
#include <type_traits>

#include "tc_pipeline.cuh"

namespace fs2 {

constexpr int TC_KB = 16;          // input channels per K-block (one K=16 FP16 MMA per split term)
constexpr int TC_CHUNKS = TC_KB / 8;  // 16-byte K-chunks (8 halfs) per K-block
constexpr int TC_SA_MAX = 8;       // activation slab stages (runtime p.SA)
constexpr int TC_SB_MAX = 8;       // weight stages (runtime p.SB)
constexpr int TC_TW = 8;            // transform warps
constexpr int TC_TTHREADS = TC_TW * 32;
constexpr int TC_CWG = 2;          // consumer warpgroups (64 output rows each)
constexpr int TC_CTHREADS = TC_CWG * 128;
constexpr int TC_THREADS = TC_CTHREADS + 32 + TC_TTHREADS + 32;   // consumer warpgroups, producer warp, transform warps, staging warp
constexpr int TC_DEPTH = 2;         // K-blocks of activation loads in flight per transform thread (register ring)
constexpr int TC_LD = 3;           // (row, K-chunk) items (2 float4 loads each) per transform thread per K-block: 256 * 3 / 2 >= 384 rows

struct TcP {
  const float* x; long long xbs, xrs;
  int B, T, Cin;
  const float* wt;                 // tiled weights, see packing.pack_conv_tc
  const float* bias;
  int N;                           // total output channels, a multiple of the kernel's NB
  int taps, dil, pad;
  int in_act; float in_slope;
  int out_act; float out_slope;
  const float* res; long long rbs, rrs;
  float alpha; int accumulate;
  const int* row_lens;
  float* y; long long ybs, yrs;
  int SA, SB;                      // ring depths
  int TPS;                         // conv taps per weight stage (small NB: several taps share one bulk copy / one handshake)
  int R;                           // slab rows held in smem (>= 128 + (taps-1)*dil, R % 8 == 4)
  int tiles_per_batch, n_items;    // work items of the padded shape: per utterance ceil(T / 128), in all (N/(NG*NB)) * B * tiles_per_batch
  int nseg;                       // K-segments per output tile (1 = plain conv).  > 1: the conv is the sum of nseg one-tap slices over p.Cin (= 256)
                                   // input channels each, slice s = (tap = s / seg_nkc, channel chunk = s % seg_nkc); every slice is its own work unit with a
                                   // fresh accumulator, and the units of one tile run back to back on one CTA, adding into y in fp32 (FS2_TC_VARIANT_SEGMENTED)
  int seg_nkc;                     // channel chunks per tap
  long long seg_wbytes;            // bytes between the tile buffers of consecutive slices
  int f8;                          // operand split: 0 = three FP16 MMAs (hi*hi + lo*hi + hi*lo), 1 = FP16 main term + ONE E4M3 (K = 32) correction MMA
  const int* x_lens;               // ragged batch (fs2_conv1d_args::x_lens) or NULL
  int lens_scale;
  int stage_off;                   // shared-memory byte offset of the staged epilogue inputs (used only if tc_stage_tiles(...) > 0)
  RowWindow win;                   // windowed mode (conv_tc_streams_kernel only): rows computed and read, see RowWindow
  const int* org;                  // the windowed mode's per-utterance origins, see origin_rows
  ModelTable table;                // table mode (conv_tc_table_kernel only): wt and bias per work item, see FieldRef
  FieldRef wt_ref, bias_ref;       // (bias stays the "has a bias" flag)
  int slot_off;                    // shared-memory byte offset of the TcSlot ring, past the plan's budget
  int NG;                          // NB-channel blocks per work item, computed one after another from the item's slab (see conv_tc_body)
};

// The weight producer decodes each unit (work item, channel block) -- its tile and block, and its model's weight-scale header and
// bias in the table mode -- into a slot of a small shared-memory ring before it pushes the unit's first weight stage, whose
// full barrier then publishes the slot to the consumers; they read it in the unit's epilogue.  So the consumer warpgroups hold no
// work-list cursor (with one, the ragged and windowed cursors' state pushes the 96-register warpgroups into spills).  The producer runs
// at most TC_SB_MAX stages, so at most TC_SB_MAX units, ahead of an epilogue: TC_SLOTS > TC_SB_MAX + 1 slots.
// The table mode's slot also carries the unit's tile base: a K-segmented conv's consumers read segment seg's weight-scale header there.
struct TcSlot { Item it; const float* bias; float inv_ws; int pad_; };
struct TcTableSlot : TcSlot { const float* wt; };
constexpr int TC_SLOTS = 16;
constexpr int TC_SLOT_BYTES = TC_SLOTS * (int)sizeof(TcSlot);
constexpr int TC_TABLE_SLOT_BYTES = TC_SLOTS * (int)sizeof(TcTableSlot);
template <class S = TcSlot>
__device__ __forceinline__ S& tc_slot(const TcP& p, unsigned char* smem, int u) {
  return reinterpret_cast<S*>(smem + p.slot_off)[u % TC_SLOTS];
}

// Shared-memory epilogue tiles behind the ring barriers: [full, empty mbarrier per consumer warp][residual tile if res][sum tile if
// accumulate or nseg > 1],
// each tile 128 rows x (NB + TC_STAGE_PAD) fp32.  The pad makes the row stride 8 or 24 banks (mod 32) for every NB, so the float2
// reads of a half warp (4 rows x 32 bytes) fall in 32 distinct banks.  The host budgets exactly these bytes (conv_tc_plan).
constexpr int TC_STAGE_PAD = 8;
constexpr int TC_RING_BAR_BYTES = (2 * TC_SA_MAX + 2 * TC_SB_MAX) * 8 + 16;
__host__ __device__ constexpr int tc_stage_tiles(bool res, bool accumulate, int nseg) { return (res ? 1 : 0) + (accumulate || nseg > 1 ? 1 : 0); }
__host__ __device__ constexpr size_t tc_stage_tile_bytes(int NB) { return (size_t)128 * (NB + TC_STAGE_PAD) * 4; }
__host__ __device__ constexpr size_t tc_stage_bytes(int NB, int tiles) { return tiles ? 2 * TC_CTHREADS / 32 * 8 + tiles * tc_stage_tile_bytes(NB) : 0; }

// 8 consecutive floats (one 32-byte sector) as two 128-bit read-only loads
__device__ __forceinline__ void ldg256(float (&d)[8], const float* src) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(src)), b = __ldg(reinterpret_cast<const float4*>(src) + 1);
  d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w; d[4] = b.x; d[5] = b.y; d[6] = b.z; d[7] = b.w;
}

template <int ACT>
__device__ __forceinline__ float tc_act(float v, float slope) {
  if (ACT == FS2_ACT_RELU) return fmaxf(v, 0.f);
  if (ACT == FS2_ACT_TANH) return tanhf(v);
  if (ACT == FS2_ACT_LRELU) return v > 0.f ? v : v * slope;
  return v;
}

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
      if (F8) {
        uint32_t l8, h8;
        hw[j] = split_f8x2(a0, a1, l8, h8);
        if (j & 1) { lw[j >> 1] |= l8 << 16; lw[2 + (j >> 1)] |= h8 << 16; }
        else { lw[j >> 1] = l8; lw[2 + (j >> 1)] = h8; }
      } else {
        hw[j] = split_f16x2(a0, a1, lw[j]);
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

// Staged-tile accesses through explicit 32-bit shared addresses (one register per row, immediate column offsets).  volatile: the
// sum tile is read back by the same thread in the next K-segment, so these stay in program order.
__device__ __forceinline__ float2 lds_f2(uint32_t a) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void sts_f2(uint32_t a, float2 v) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a), "f"(v.x), "f"(v.y) : "memory");
}

// The staged region (TcP::stage_off bytes into shared memory): per consumer warp a `full` and an `empty` mbarrier, then the tiles.
// Addresses are recomputed from the kernel parameters where they are used: the consumer warps are at their register cap.
template <int NB>
struct TcStage {
  static constexpr int CWARPS = TC_CTHREADS / 32;
  static __device__ __forceinline__ uint64_t* full(const TcP& p, unsigned char* smem, int warp) {
    return reinterpret_cast<uint64_t*>(smem + p.stage_off) + warp;
  }
  static __device__ __forceinline__ uint64_t* empty(const TcP& p, unsigned char* smem, int warp) { return full(p, smem, warp) + CWARPS; }
  static __device__ __forceinline__ float* res_tile(const TcP& p, unsigned char* smem) {
    return reinterpret_cast<float*>(smem + p.stage_off + 2 * CWARPS * 8);
  }
  static __device__ __forceinline__ float* sum_tile(const TcP& p, unsigned char* smem) {
    return res_tile(p, smem) + (p.res ? tc_stage_tile_bytes(NB) / 4 : 0);
  }
  // Staging warp, channel block it.nblk of a work item: for each consumer warp w, once w has released its rows of the previous block, bulk-copy
  // the residual / old y rows of its 16 tile rows below it.rows (one copy per row and tile), completing on full[w].  `phase`: parity of
  // this CTA's (item, block) count.
  static __device__ __forceinline__ void fill(const TcP& p, unsigned char* smem, const Item& it, uint32_t phase) {
    const int lane = threadIdx.x & 31;
    const uint32_t row_bytes = NB * 4, per_row = (p.res ? row_bytes : 0u) + (p.accumulate ? row_bytes : 0u);
    for (int w = 0; w < CWARPS; w++) {
      const int row0 = 16 * w, rows = max(0, min(16, it.rows - (it.t0 + row0)));
      mbar_wait(empty(p, smem, w), phase ^ 1u);
      if (lane == 0) mbar_expect_tx(full(p, smem, w), (uint32_t)rows * per_row);
      __syncwarp();
      if (lane < rows) {
        const long long t = it.t0 + row0 + lane;
        const int srow = (row0 + lane) * (NB + TC_STAGE_PAD), n0 = it.nblk * NB;
        if (p.res) bulk_g2s(res_tile(p, smem) + srow, p.res + it.b * p.rbs + t * p.rrs + n0, row_bytes, full(p, smem, w));
        if (p.accumulate) bulk_g2s(sum_tile(p, smem) + srow, p.y + it.b * p.ybs + t * p.yrs + n0, row_bytes, full(p, smem, w));
      }
      __syncwarp();
    }
  }
};

// Epilogue of one consumer warpgroup: its 64 rows of the tile straight from the accumulator fragments (see wgmma.cuh): thread
// (warp w, lane l) owns rows 16w + l/4 and +8, column pairs 8j + 2(l%4).  The split-term accumulators are summed here in fp32
// round-to-nearest.  bias / row_lens may be NULL.  The residual and the value to accumulate come from row t - t0 of the staged tiles
// (TcStage): use_res adds the residual tile; sum_in adds alpha*value to the sum tile's value instead of overwriting it; the result goes to
// y, or with sum_out to the sum tile (a K-segmented slice before the last).  Rows >= it.rows (T, or n_b of a ragged batch) are not written.
// The tiles are addressed through 32-bit shared addresses derived from the kernel parameters (the kernel is at its 96-register cap).
template <int ACT, int NB, int TG>
__device__ __forceinline__ void tc_epilogue(const TcP& p, float (&acc)[TG][NB / 2], const Item& it, int row_base, const float* bias,
                                            const int* row_lens, unsigned char* smem, bool use_res, bool sum_in, bool sum_out, float inv_ws) {
  const int lane = threadIdx.x & 31;
  const int n0 = it.nblk * NB + 2 * (lane & 3);
  const int len_b = row_lens ? min(row_lens[it.b], p.T) : p.T;
  const float slope = p.out_slope, alpha = p.alpha;
  const float* brow = bias ? bias + n0 : nullptr;      // one base, immediate column offsets
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int t = row_base + (lane >> 2) + 8 * h;
    if (t >= it.rows) continue;
    const bool live = t < len_b;
    float* yrow = p.y + (long long)it.b * p.ybs + (long long)t * p.yrs + n0;
    // shared address of this thread's first column in the residual tile; the sum tile follows it when there is a residual
    const uint32_t sres = smem_u32(TcStage<NB>::res_tile(p, smem)) + 4u * ((t - it.t0) * (NB + TC_STAGE_PAD) + 2 * (lane & 3));
    const uint32_t ssum = sres + (p.res ? (uint32_t)tc_stage_tile_bytes(NB) : 0u);
#pragma unroll
    for (int j = 0; j < NB / 8; j++) {
      float a0 = acc[0][4 * j + 2 * h], a1 = acc[0][4 * j + 2 * h + 1];
      if (TG == 2) { a0 += acc[TG - 1][4 * j + 2 * h]; a1 += acc[TG - 1][4 * j + 2 * h + 1]; }
      float2 bv = make_float2(0.f, 0.f);
      if (brow) bv = __ldg(reinterpret_cast<const float2*>(brow + 8 * j));
      float2 o;
      o.x = tc_act<ACT>(fmaf(a0, inv_ws, bv.x), slope);    // inv_ws is a power of two: exact
      o.y = tc_act<ACT>(fmaf(a1, inv_ws, bv.y), slope);
      if (use_res) {
        const float2 rv = lds_f2(sres + 32 * j);
        o.x += rv.x; o.y += rv.y;
      }
      if (sum_in) {
        const float2 yv = lds_f2(ssum + 32 * j);
        o.x = o.x * alpha + yv.x; o.y = o.y * alpha + yv.y;
      } else {
        o.x *= alpha; o.y *= alpha;
      }
      if (!live) o = make_float2(0.f, 0.f);
      if (sum_out) sts_f2(ssum + 32 * j, o);
      else *reinterpret_cast<float2*>(yrow + 8 * j) = o;
    }
  }
}

// RAG: ragged batch (TcP::x_lens != NULL), see WorkList (every NB is at or near the 96-register cap of one 544-thread CTA per SM).
// WIN: windowed mode with per-utterance origins, see WindowList and origin_rows: the tiles start at p.win.y0, rows at or beyond
// p.win.yend are not written and rows at or beyond p.win.xend are not read (the host biases x, res and y by the window origins, so rows
// are window rows here), and utterance b's rows outside [lo_b, hi_b) read as zero.
// TABLE: table mode: each work item reads the tiles, weight-scale headers and bias of its utterance's model (p.table), loaded once
// per item instead of once per CTA, K-segmented convs included.
template <int NB, bool RAG, bool WIN, bool TABLE = false>
__device__ __forceinline__ void conv_tc_body(const TcP& p) {
  constexpr int TG = NB <= 64 ? 2 : 1;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = warp_uniform_id(), lane = tid & 31;
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
  const bool staged = tc_stage_tiles(p.res != nullptr, p.accumulate != 0, p.nseg) > 0;   // the host budgeted tc_stage_bytes
  using Stage = TcStage<NB>;
  using Slot = std::conditional_t<TABLE, TcTableSlot, TcSlot>;

  const int KBLOCKS = p.Cin / TC_KB;
  constexpr int CWARPS = TC_CTHREADS / 32;
  const int NG = p.NG;
  // 128-row tiles x NB-channel blocks; windowed: item.rows bounds the stores, the transform warps bound their loads at min(hi_b, xend)
  std::conditional_t<WIN, WindowList, WorkList<RAG>> work;
  if constexpr (WIN) work.init(p.x_lens, p.org, p.lens_scale, p.B, 128, p.n_items / (p.B * p.tiles_per_batch), p.win.y0, p.win.yend, p.win.yend);
  else work.init(p.x_lens, p.lens_scale, p.T, p.B, 128, p.tiles_per_batch, p.n_items);

  if (tid == 0) {
    ring_init(fullA, emptyA, TC_SA_MAX, TC_TW, CWARPS);
    ring_init(fullB, emptyB, TC_SB_MAX, 1, CWARPS);
    if (staged) ring_init(Stage::full(p, smem_raw, 0), Stage::empty(p, smem_raw, 0), CWARPS, 1, 1);
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == CWARPS) {
    // ===================== weight-stage producer (TMA bulk copies) =====================
    if (lane == 0) {
      const uint32_t stage_bytes = 2 * b_plane;   // one tap of one K-block (hi + lo)
      Ring rb;
      const float inv_ws0 = __ldg(p.wt);               // header: 1 / (power-of-two weight scale)
      for (int item = blockIdx.x, u = 0; item < work.count; item += gridDim.x) {
        const Item pit = work.item(item);
        const float* wt = p.wt;
        const float* bias = p.bias;
        float inv_ws = inv_ws0;
        if constexpr (TABLE) {                         // the item's model's
          wt = row_weight(p.table, pit.b, p.wt_ref);
          bias = p.bias ? row_weight(p.table, pit.b, p.bias_ref) : nullptr;
          inv_ws = __ldg(wt);
        }
        for (int j = 0; j < NG; j++, u++) {            // the item's blocks, in the consumers' order
          Slot& slot = tc_slot<Slot>(p, smem_raw, u);   // before the unit's first stage: its full barrier publishes the slot
          slot.it = Item{pit.nblk * NG + j, pit.b, pit.t0, pit.rows};
          slot.bias = bias;
          slot.inv_ws = inv_ws;
          if constexpr (TABLE) slot.wt = wt;
          for (int seg = 0; seg < p.nseg; seg++) {
            const unsigned char* src = reinterpret_cast<const unsigned char*>(wt) + (long long)seg * p.seg_wbytes + TC_HDR +
                                       (size_t)slot.it.nblk * p.taps * KBLOCKS * stage_bytes;   // tiles are ordered [kb][tap]
            for (int kb = 0; kb < KBLOCKS; kb++) {
              for (int tap = 0; tap < p.taps; tap += p.TPS) {
                const uint32_t bytes = (uint32_t)min(p.TPS, p.taps - tap) * stage_bytes;
                ring_push(fullB, emptyB, rb, SB, b_base + (size_t)rb.idx * p.TPS * stage_bytes, src, bytes);
                src += bytes;
              }
            }
          }
        }
      }
    }
  } else if (warp < CWARPS) {
    // ===================== consumer warpgroups: MMAs + epilogue =====================
    // Every operand is a precomputed descriptor base plus a constant.
    const int g = warp >> 2;                             // 64-row half of the tile
    const uint64_t a_const = wgmma_desc(0, (uint32_t)R * 16, 128), b_const = wgmma_desc(0, (uint32_t)NB * 16, 128);
    Ring ra, rb;
    // This CTA's units (work item, channel block): the item's NG blocks one after another, each a full pass over the item's slab stages
    // (NG > 1: nseg == 1 and SA >= KBLOCKS, planned on the host).  Every pass but the last rewinds the slab cursor and keeps the stages
    // full.  The unit's tile and block come from the producer's slot (TcSlot).
    const int units = (work.count - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x * NG;
    for (int unit = 0, blk = 0; unit < units; unit++, blk = blk == NG - 1 ? 0 : blk + 1) {   // blk: the unit's block in its item
      const bool last_pass = blk == NG - 1;
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
            const int n = min(p.TPS, p.taps - tap);
            ring_step(fullB, emptyB, rb, pend_b, [&](uint32_t sb) {
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
            });
            ring_release_last(emptyA, pend_a, last_pass);   // its last group retired in ring_step
          }
          pend_a = (int)sa;
        }
        wgmma_wait<0>();
#pragma unroll
        for (int gg = 0; gg < TG; gg++) wgmma_keep<NB>(acc[gg]);
        if (pend_b >= 0) tc_release(&emptyB[pend_b]);
        ring_release_last(emptyA, pend_a, last_pass);
        if (!last_pass) ra.rewind(SA, KBLOCKS);
        // K-segmented conv: unit (item, seg) adds slice seg of the tile into the sum tile -- bias with the first slice; residual,
        // alpha-free sum, the pad-row mask and the store to y with the last.  The same thread owns the same outputs in every unit, so the
        // fp32 read-modify-write of the sum tile needs no further ordering.  No output activation (checked on the host).
        const bool first = seg == 0, last = seg == p.nseg - 1;
        const Slot& slot = tc_slot<Slot>(p, smem_raw, unit);
        const Item it = slot.it;
        // the staging barrier completes one phase per unit of this CTA
        if (staged && first) mbar_wait(Stage::full(p, smem_raw, warp), (uint32_t)unit & 1u);
        const float* bias = first ? slot.bias : nullptr;
        const int* lens = last ? p.row_lens : nullptr;
        const bool use_res = last && p.res, sum_in = !first || p.accumulate, sum_out = !last;
        // header: 1 / (power-of-two weight scale) of the unit's model; a K-segmented conv's segment seg has its own
        const float* hdr = p.wt;
        if constexpr (TABLE) hdr = slot.wt;
        const float inv_ws = p.nseg == 1 ? slot.inv_ws
            : __ldg(reinterpret_cast<const float*>(reinterpret_cast<const unsigned char*>(hdr) + (long long)seg * p.seg_wbytes));
        const int row_base = it.t0 + 64 * g + 16 * (warp & 3);
        switch (p.out_act) {                           // uniform branch: keeps tanhf out of the other variants' inner loops
          case FS2_ACT_RELU: tc_epilogue<FS2_ACT_RELU, NB, TG>(p, acc, it, row_base, bias, lens, smem_raw, use_res, sum_in, sum_out, inv_ws); break;
          case FS2_ACT_TANH: tc_epilogue<FS2_ACT_TANH, NB, TG>(p, acc, it, row_base, bias, lens, smem_raw, use_res, sum_in, sum_out, inv_ws); break;
          case FS2_ACT_LRELU: tc_epilogue<FS2_ACT_LRELU, NB, TG>(p, acc, it, row_base, bias, lens, smem_raw, use_res, sum_in, sum_out, inv_ws); break;
          default: tc_epilogue<FS2_ACT_NONE, NB, TG>(p, acc, it, row_base, bias, lens, smem_raw, use_res, sum_in, sum_out, inv_ws); break;
        }
      }
      if (staged) {                                    // this warp's rows are read: the staging warp may refill them
        fence_proxy_async();                           // this lane's generic reads / writes of the rows -> before the bulk copies
        tc_release(Stage::empty(p, smem_raw, warp));
      }
    }
  } else if (warp == TC_THREADS / 32 - 1) {
    // ===================== staging warp: residual / old-y rows of each work item and block -> shared memory (TcStage) ================
    if (staged) {
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < work.count; item += gridDim.x) {
        const Item it = work.item(item);
        for (int j = 0; j < NG; j++, phase ^= 1u) Stage::fill(p, smem_raw, Item{it.nblk * NG + j, it.b, it.t0, it.rows}, phase);
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
    int l_tlo = 0;                                     // rows below it read as zero: 0, or lo_b in the windowed mode
    bool l_interior = false;                           // warp-uniform: every slab row of the item exists
    auto l_set_item = [&]() {
      if (l_item < work.count) {
        const Item it = work.item(l_item);
        if constexpr (WIN) l_tend = work.rows_of(it.b, p.win.xend);
        else l_tend = it.rows;
        if constexpr (WIN) l_tlo = work.lo_of(it.b);
        const int s_tap = l_seg / p.seg_nkc, s_kc = l_seg - s_tap * p.seg_nkc;   // K-segment: one tap, one 256-channel chunk (0, 0 when nseg == 1)
        l_tfirst = it.t0 - p.pad + s_tap;
        l_xrow = p.x + (long long)it.b * p.xbs + (long long)l_tfirst * p.xrs + s_kc * p.Cin;
        if constexpr (WIN) l_interior = l_tfirst >= l_tlo && l_tfirst + rows_needed <= l_tend;
        else l_interior = l_tfirst >= 0 && l_tfirst + rows_needed <= l_tend;
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
          bool in;
          if constexpr (WIN) in = rowu[u] >= 0 && t >= l_tlo && t < l_tend;
          else in = rowu[u] >= 0 && t >= 0 && t < l_tend;
          if (in) {
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
    const int my_items = (work.count - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // >= 0: blockIdx.x < gridDim.x
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
          tc_release(&fullA[ra.idx]);                  // one arrival per transform warp
          ra.advance(SA);
          if (seq + DEPTH < total) issue_loads(v[d]);
        }
      }
    }
  }
}

template <int NB, bool RAG>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const TcP p) {
  conv_tc_body<NB, RAG, false>(p);
}

// Windowed mode (fs2_vocoder_forward_window and _streams): an entry point of its own, so that the padded and ragged instantiations keep
// their code (p.org and the lens are not NULL here).
template <int NB>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_streams_kernel(const TcP p) {
  conv_tc_body<NB, true, true>(p);
}

// Table mode (ModelTable): the windowed conv (multi-generator pool) or the offline padded or ragged one (voices) with each item's
// weights from its utterance's model
template <int NB, bool RAG, bool WIN>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_table_kernel(const TcP p) {
  conv_tc_body<NB, RAG, WIN, true>(p);
}

// The NB instantiations live in their own translation units (conv_tc_nb*.cu) so that the library builds in parallel.
// conv_tc_prepare_nb / conv_tc_launch_nb return cudaErrorInvalidValue for an NB they do not instantiate.  The entry point follows from
// the mode: window (the windowed mode), p.table.models (the table mode) and p.x_lens (a ragged offline batch).
#define FS2_CONV_TC_NB_DECL(nb)                        \
  cudaError_t conv_tc_prepare_nb##nb(int smem_bytes); \
  void conv_tc_launch_nb##nb(const TcP& p, bool window, unsigned grid, size_t smem, cudaStream_t s);
FS2_CONV_TC_NB_DECL(16) FS2_CONV_TC_NB_DECL(32) FS2_CONV_TC_NB_DECL(48) FS2_CONV_TC_NB_DECL(64)
FS2_CONV_TC_NB_DECL(80) FS2_CONV_TC_NB_DECL(96) FS2_CONV_TC_NB_DECL(112) FS2_CONV_TC_NB_DECL(128)
#undef FS2_CONV_TC_NB_DECL

#define FS2_CONV_TC_NB_DEF(nb)                                                                                            \
  cudaError_t conv_tc_prepare_nb##nb(int smem_bytes) {                                                                    \
    cudaError_t e = cudaSuccess;                                                                                          \
    for (const void* k : {(const void*)conv_tc_kernel<nb, false>, (const void*)conv_tc_kernel<nb, true>,                   \
                          (const void*)conv_tc_streams_kernel<nb>, (const void*)conv_tc_table_kernel<nb, false, false>,    \
                          (const void*)conv_tc_table_kernel<nb, true, false>, (const void*)conv_tc_table_kernel<nb, true, true>}) \
      if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);        \
    return e;                                                                                                             \
  }                                                                                                                       \
  void conv_tc_launch_nb##nb(const TcP& p, bool window, unsigned grid, size_t smem, cudaStream_t s) {                     \
    void (*k)(const TcP);                                                                                                 \
    if (p.table.models) k = window ? conv_tc_table_kernel<nb, true, true>                                                 \
                            : p.x_lens ? conv_tc_table_kernel<nb, true, false> : conv_tc_table_kernel<nb, false, false>;    \
    else k = window ? conv_tc_streams_kernel<nb> : p.x_lens ? conv_tc_kernel<nb, true> : conv_tc_kernel<nb, false>;       \
    k<<<grid, TC_THREADS, smem, s>>>(p);                                                                                  \
  }

}  // namespace fs2
