// Device code shared by the warp-specialised wgmma kernels of conv_tc_kernel.cuh, resstack_fused.cu and attention_fused.cu.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace fs2 {

constexpr int TC_HDR = 128;        // bytes of header in front of the weight tiles: float[0] = 1 / weight scale

// Operand scales of the f16 + f8 split (TcP::f8): activation lo * 2^12 and hi (unscaled) are rounded to E4M3; the packer stores
// weight hi * 2^-12 and lo (unscaled) in E4M3 (packing.pack_conv_tc), so both correction products carry the main term's scale.
// lo * 2^12 stays inside E4M3 for |x| < 256 and hi for |x| <= 448; beyond that the correction of that element saturates (the result
// degrades towards single-pass fp16 accuracy for it, never to garbage).
constexpr float TC_F8_LO_SCALE = 4096.f;
constexpr float TC_F8_HI_SCALE = 1.f;

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

// Operand split of {a0, a1}: returns hi = fp16(a) as fp16x2 and stores lo = fp16(a - hi) the same way (a - hi is exact in fp32).
__device__ __forceinline__ uint32_t split_f16x2(float a0, float a1, uint32_t& lo) {
  const uint32_t hi = cvt_f16x2_sat(a0, a1);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo = cvt_f16x2_sat(a0 - hf.x, a1 - hf.y);
  return hi;
}

// The f16 + f8 split: hi as above, and the E4M3 pairs lo8 = e4m3((a - hi) * TC_F8_LO_SCALE), hi8 = e4m3(hi * TC_F8_HI_SCALE).
__device__ __forceinline__ uint32_t split_f8x2(float a0, float a1, uint32_t& lo8, uint32_t& hi8) {
  static_assert(TC_F8_HI_SCALE == 1.f, "hi8 is hi rounded to E4M3 unscaled");
  const uint32_t hi = cvt_f16x2_sat(a0, a1);
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  lo8 = cvt_e4m3x2_sat((a0 - hf.x) * TC_F8_LO_SCALE, (a1 - hf.y) * TC_F8_LO_SCALE);
  hi8 = cvt_e4m3x2_sat(hf.x, hf.y);
  return hi;
}

// Warp index of the calling thread, in a form ptxas knows to be warp-uniform.  threadIdx.x >> 5 is uniform only because the
// block is one-dimensional, which ptxas cannot assume: a role branch on it counts as divergent, and every wgmma under such a
// branch is then serialised (warning C7520: a warpgroup arrive and a full wait around each MMA, so commit groups and
// wait_group<1> stop overlapping anything).  A shuffle from lane 0 is uniform by construction.
__device__ __forceinline__ int warp_uniform_id() { return __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0); }

// ------------------------------------------------------------------ stage ring
// n shared-memory stages with a `full` and an `empty` mbarrier each; every role walks the same stage sequence with its own cursor.
// mbarrier ring cursor without runtime div/mod (an integer division per tap was on the MMA issuer's critical path)
struct Ring {
  uint32_t idx = 0, phase = 0;
  __device__ __forceinline__ void advance(uint32_t n) {
    if (++idx == n) { idx = 0; phase ^= 1u; }
  }
  // back over the last `steps` <= n stages: the next pass of a consumer that reads them more than once (ring_release_last)
  __device__ __forceinline__ void rewind(uint32_t n, uint32_t steps) {
    if (idx < steps) { idx += n; phase ^= 1u; }
    idx -= steps;
  }
};

// One thread initialises the barrier pairs of an n-stage ring; mbar_init_fence() then orders every init before the barriers' use.
__device__ __forceinline__ void ring_init(uint64_t* full, uint64_t* empty, int n, int full_count, int empty_count) {
  for (int i = 0; i < n; i++) { mbar_init(&full[i], full_count); mbar_init(&empty[i], empty_count); }
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// Producer: waits until the cursor's stage is free, then fills `bytes` of it at dst with one bulk copy from global src.
__device__ __forceinline__ void ring_push(uint64_t* full, uint64_t* empty, Ring& r, uint32_t n, void* dst, const void* src, uint32_t bytes) {
  mbar_wait(&empty[r.idx], r.phase ^ 1);
  mbar_expect_tx(&full[r.idx], bytes);
  bulk_g2s(dst, src, bytes, &full[r.idx]);
  r.advance(n);
}

// One arrival per warp once all its lanes are done with a stage (a consumer's MMAs have retired, or a producer's stores are complete).
__device__ __forceinline__ void tc_release(uint64_t* bar) {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) mbar_arrive(bar);
}

// Consumer warpgroup: waits for the cursor's stage, issues mmas(stage) as one wgmma group and releases the previous group's stage
// once that has retired (so the next stage's MMAs are always queued).  pend: the last group's stage, -1 before the first step.  The
// caller advances the cursor after the step, once it has also released what else the previous group read (the conv's slab).
template <class Mmas>
__device__ __forceinline__ void ring_step(uint64_t* full, uint64_t* empty, const Ring& r, int& pend, Mmas&& mmas) {
  mbar_wait(&full[r.idx], r.phase);
  wgmma_fence();
  mmas(r.idx);
  wgmma_commit();
  wgmma_wait<1>();
  if (pend >= 0) tc_release(&empty[pend]);
  pend = (int)r.idx;
}

// Consumer that reads a span of stages in several passes (the conv's slab: once per channel block of a work item): pend, a stage whose
// reads have retired, is released only on the last pass, so the producer cannot refill it while a later pass still needs it; earlier
// passes find it still full (the same phase) after Ring::rewind.  The ring needs at least as many stages as the span.
__device__ __forceinline__ void ring_release_last(uint64_t* empty, int& pend, bool last) {
  if (pend >= 0 && last) tc_release(&empty[pend]);
  pend = -1;
}

// After at least one ring_step: waits for every wgmma group and releases the last stage; then wgmma_keep the accumulators.
__device__ __forceinline__ void ring_drain(uint64_t* empty, int pend) { wgmma_wait<0>(); tc_release(&empty[pend]); }

// ------------------------------------------------------------------ work list
// One work item: block nblk (of output channels; of heads in attention), utterance b, first row t0 of its `tile` rows, and the rows
// of utterance b that exist (the padded length cap, or n_b of a ragged batch): rows >= `rows` are padding.
struct Item { int nblk, b, t0, rows; };

// The work list of a persistent kernel: blocks x B utterances x `tile`-row tiles, items ordered (block, utterance, tile).  Every role
// of a CTA walks it as  for (i = blockIdx.x; i < count; i += gridDim.x) { const Item it = work.item(i); ... }  with its own copy, so
// all roles see the same item sequence: the mbarrier rings only work if they do.
// init's per_b = ceil(cap / tile) and items = blocks * B * per_b are the padded shape's tiles per utterance and item count as the host
// planned them: as kernel parameters they cost the padded instantiations no registers, computed here they did.
// RAG: ragged batch (lens != NULL): utterance b has n_b = ragged_rows(lens, scale, cap, b) rows and only its live tiles are items,
// sum_b ceil(n_b / tile) per block, so no tile lying wholly in the padding is ever scheduled.  MIN_ROWS > 0: an utterance with fewer
// rows counts as empty (the fused attention kernel leaves those to the exact one).  RAG is a template parameter rather than a runtime
// branch: the cursor state would otherwise cost the padded instantiations registers.
template <bool RAG, int MIN_ROWS = 0>
struct WorkList;

// Padded batch: every utterance has cap rows, and an item index decodes by plain division.
template <int MIN_ROWS>
struct WorkList<false, MIN_ROWS> {
  int count, B, tile, cap, per_b;
  __device__ __forceinline__ void init(const int*, int, int cap_, int B_, int tile_, int per_b_, int items) {
    cap = cap_; B = B_; tile = tile_; per_b = per_b_; count = items;
  }
  __device__ __forceinline__ Item item(int i) const {
    const int per_blk = B * per_b;
    Item it;
    it.nblk = i / per_blk;
    const int rem = i - it.nblk * per_blk;
    it.b = rem / per_b;
    it.t0 = (rem - it.b * per_b) * tile;
    it.rows = cap;
    return it;
  }
};

// Ragged batch: a monotone cursor over the compacted sequence.  A role visits its items in increasing order, so the cursor only moves
// forward and each length is loaded once per block: no table, no cap on B, no host sync.
template <int MIN_ROWS>
struct WorkList<true, MIN_ROWS> {
  const int* lens; int scale, cap, tile;
  int count, live;                 // items; live tiles per block
  int nblk, b, before, rows;       // cursor: block, utterance, live tiles of utterances < b in the block, n_b
  __device__ __forceinline__ int rows_of(int u) const {
    const int n = ragged_rows(lens, scale, cap, u);
    if constexpr (MIN_ROWS > 0) return n < MIN_ROWS ? 0 : n;
    return n;
  }
  __device__ __forceinline__ void init(const int* lens_, int scale_, int cap_, int B, int tile_, int per_b, int items) {
    lens = lens_; scale = scale_; cap = cap_; tile = tile_;
    live = 0;
    for (int u = 0; u < B; u++) live += (rows_of(u) + tile - 1) / tile;
    count = live * (items / (B * per_b));          // live tiles x blocks
    nblk = 0; b = 0; before = 0; rows = rows_of(0);
  }
  __device__ __forceinline__ Item item(int i) {   // i < count, and not below the previous call's i
    const int blk = i / live, rem = i - blk * live;
    if (blk != nblk) { nblk = blk; b = 0; before = 0; rows = rows_of(0); }
    for (int nt = (rows + tile - 1) / tile; rem >= before + nt; nt = (rows + tile - 1) / tile) {
      before += nt;
      rows = rows_of(++b);
    }
    Item it;
    it.nblk = blk; it.b = b; it.t0 = (rem - before) * tile; it.rows = rows;
    return it;
  }
};

// Windowed mode, per-utterance origins (origin_rows; fs2_vocoder_forward_window and _streams): only the window rows [y0, yend) are
// computed, in `tile`-row tiles that start at y0.  Utterance b's rows are [lo_b, hi_b) of the window buffers; only the tiles that
// overlap [max(y0, lo_b), min(yend, hi_b)) are items, and the tile grid still starts at y0, so every utterance's tiles cover the same
// window rows and every role walks the same monotone item sequence.  An item's t0 is its tile's first window row and its `rows` is
// min(hi_b, lim), lim >= yend: the bound of the rows the kernel stores (conv_tc), or the layer's length (resstack, whose tensor maps
// bound its loads and stores); rows_of(b, end) gives another, lo_of(b) gives lo_b.  The cursor is the ragged one's.
struct WindowList {
  const int* lens; const int* org; int scale, tile, y0, yend, lim;
  int count, live;
  int nblk, b, before, rows, first;   // cursor; rows = min(hi_b, lim), first = utterance b's first live tile
  __device__ __forceinline__ int rows_of(int u, int end) const { return min(origin_rows(lens, org, scale, u).hi, end); }
  __device__ __forceinline__ int rows_of(int u) const { return rows_of(u, lim); }
  __device__ __forceinline__ int lo_of(int u) const { return origin_rows(lens, org, scale, u).lo; }
  __device__ __forceinline__ int first_of(int u) const { return max(0, lo_of(u) - y0) / tile; }
  __device__ __forceinline__ int tiles_of(int r, int f) const { return max(0, max(0, min(r, yend) - y0 + tile - 1) / tile - f); }
  __device__ __forceinline__ void init(const int* lens_, const int* org_, int scale_, int B, int tile_, int blocks, int y0_, int yend_,
                                       int lim_) {
    lens = lens_; org = org_; scale = scale_; tile = tile_; y0 = y0_; yend = yend_; lim = lim_;
    live = 0;
    for (int u = 0; u < B; u++) live += tiles_of(rows_of(u), first_of(u));
    count = live * blocks;
    nblk = 0; b = 0; before = 0; rows = rows_of(0); first = first_of(0);
  }
  __device__ __forceinline__ Item item(int i) {   // i < count, and not below the previous call's i
    const int blk = i / live, rem = i - blk * live;
    if (blk != nblk) { nblk = blk; b = 0; before = 0; rows = rows_of(0); first = first_of(0); }
    for (int nt = tiles_of(rows, first); rem >= before + nt; nt = tiles_of(rows, first)) {
      before += nt;
      rows = rows_of(++b);
      first = first_of(b);
    }
    Item it;
    it.nblk = blk; it.b = b; it.t0 = y0 + (first + rem - before) * tile; it.rows = rows;
    return it;
  }
};

}  // namespace fs2
