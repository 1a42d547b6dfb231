// Fused self-attention of one FFT block on the tensor cores (transformer/Modules.py:14-25 + key mask Models.py:79, heads as
// SubLayers.py:39-44): S = Q K^T, softmax and O = P V in ONE persistent wgmma kernel -- the score matrix lives in registers and
// never reaches HBM (the reference writes S [2B][T][T] in fp32 four times).
//
//   pack_kv_tiles_kernel, once per layer: K and V of every (utterance, head) x AF_WSCALE -> fp16 hi/lo operand tiles, one bulk-copy
//   stage per 16 rows of the MMA's K dimension.  Every MMA is the three-MMA split (DESIGN §3): 22 significant bits per operand while its
//   lo part is a normal fp16 number, and an absolute floor below that -- 2^-25 for Q (split unscaled), 2^-29 for K and V (x 16), about
//   2^-40 for P (x AF_PSCALE).  The converts saturate: the domain is |q| < 65504 and |k|, |v| < 4094, with no error beyond it.
//   work item = (head h, utterance b, 128 query rows).
//   pass 1: for every block of 128 keys  S = Q K_j^T (register accumulators)  ->  row maximum (a row's columns are spread over the
//           four lanes of a quad: two shuffles).
//   pass 2: S again -> p = exp2(s*c - m) (keys >= key_len masked to 0) -> fp16 hi/lo operand planes in shared memory ->
//           O += P V_j (register accumulators), row sums alongside.  No rescaling of O is ever needed because the maximum is final.
//   epilogue: O / l -> ctx[b, t, h*128 .. +128]; query rows t >= key_len[b] are written as 0 (contract of fs2_attention).
//   Recomputing S costs 1/3 more MMAs than a one-pass online softmax and removes the O rescaling.
//
// Ragged mode (template parameter RAG; the padded instantiation keeps its code): utterance b is computed exactly as a B = 1 call
// with T = n_b = key_lens[b].  Only utterances with n_b >= AF_MIN_ROWS are taken (a B = 1 call with a shorter T runs the exact
// kernel, which takes the others); their work items are the live query tiles, compacted per head by the WorkList cursor
// (tc_pipeline.cuh), and each streams ceil(n_b / 128) key blocks in both passes.  The packer packs only those key blocks, with rows at
// or beyond n_b as zero; Q rows at or beyond n_b load as zero (0 * a stale NaN would still be NaN in P V), and ctx rows there are
// not written.
//
// Roles: warp 8 streams K / V stages (cp.async.bulk) in the order they are consumed; warps 0-7 are two consumer warpgroups that
// own 64 query rows each: Q conversion, the MMAs, both softmax passes and the epilogue.
#include "tc_pipeline.cuh"

namespace fs2 {

constexpr int AF_THREADS = 288;
constexpr int AF_SB = 8;                         // K / V stage ring depth
constexpr uint32_t AF_STAGE = 8192;              // one stage: [hi | lo][2 chunks][128][16 B]
constexpr float AF_WSCALE = 16.f;                // power-of-two operand scale of the packed K / V tiles (|k|, |v| < 4094 stay inside fp16)
constexpr float AF_PSCALE = 32768.f;             // scale of p in (0, 1] before its split: lo stays normal down to p ~ 2^-18 (max 32768)
constexpr int AF_MIN_ROWS = 128;                 // shortest utterance the ragged kernel takes (a B = 1 call takes T >= 128)

// ------------------------------------------------------------------ K / V operand tiles
// Per (utterance, head) one buffer of af_tile_stride(Tk) bytes: TC_HDR header (float 1 / AF_WSCALE), then the stages; keys are padded
// to Tk, a multiple of 128, with zeros.
__device__ __forceinline__ void split8(const float (&f)[8], float scale, uint4& hi, uint4& lo) {
  uint32_t hw[4], lw[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const float a0 = fminf(fmaxf(f[2 * j] * scale, -65504.f), 65504.f);   // also maps NaN to -65504
    const float a1 = fminf(fmaxf(f[2 * j + 1] * scale, -65504.f), 65504.f);
    hw[j] = split_f16x2(a0, a1, lw[j]);
  }
  hi = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  lo = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

// K tiles: B operand W[c = d][n = key] of S = Q K^T, layout  header | [key/128][d/16][hi|lo][2 chunks][128 keys][8 halfs]
// Ragged: keys of utterance b at or beyond n_b pack as zero, and key blocks beyond ceil(n_b / 128) (every block when n_b < AF_MIN_ROWS)
// are not packed: the attention kernel never reads them.
template <bool RAG>
__device__ __forceinline__ int af_key_rows(const int* key_lens, int T, int b) {
  if (!RAG) return T;
  const int n = ragged_rows(key_lens, 1, T, b);
  return n < AF_MIN_ROWS ? 0 : n;
}

template <bool RAG>
__device__ __forceinline__ void pack_k_tiles(const float* __restrict__ qkv, unsigned char* __restrict__ tiles, int B, int T, int Tk, int H,
                                             long long tile_stride, long long idx, const int* key_lens) {   // idx = (bh, key, dchunk)
  const long long total = (long long)B * H * Tk * (128 / 8);
  if (idx >= total) return;
  const int dchunk = (int)(idx % (128 / 8));
  const long long r = idx / (128 / 8);
  const int key = (int)(r % Tk);
  const int bh = (int)(r / Tk);
  const int b = bh / H, h = bh - b * H;
  const int D = H * 128;
  const int rows = af_key_rows<RAG>(key_lens, T, b);
  if (RAG && key >= (rows + 127) / 128 * 128) return;
  float f[8];
#pragma unroll
  for (int j = 0; j < 8; j++) f[j] = 0.f;
  if (key < rows) {
    const float4* src = reinterpret_cast<const float4*>(qkv + ((long long)b * T + key) * 3 * D + D + h * 128 + dchunk * 8);
    const float4 u = __ldg(src), v = __ldg(src + 1);
    f[0] = u.x; f[1] = u.y; f[2] = u.z; f[3] = u.w; f[4] = v.x; f[5] = v.y; f[6] = v.z; f[7] = v.w;
  }
  uint4 hi, lo;
  split8(f, AF_WSCALE, hi, lo);
  unsigned char* base = tiles + (long long)bh * tile_stride;
  if (key == 0 && dchunk == 0) *reinterpret_cast<float*>(base) = 1.f / AF_WSCALE;
  const int nblk = key / 128, nn = key - nblk * 128, kb = dchunk >> 1, chunk = dchunk & 1;
  const size_t b_plane = AF_STAGE / 2, kbl = 128 / 16;
  unsigned char* dst = base + TC_HDR + ((size_t)nblk * kbl + kb) * AF_STAGE + ((size_t)chunk * 128 + nn) * 16;
  *reinterpret_cast<uint4*>(dst) = hi;
  *reinterpret_cast<uint4*>(dst + b_plane) = lo;
}

// V tiles: B operand W[c = key][n = d] of O = P V, layout  header | [key/16][hi|lo][2 chunks of 8 keys][128 d][8 halfs (keys)]
template <bool RAG>
__device__ __forceinline__ void pack_v_tiles(const float* __restrict__ qkv, unsigned char* __restrict__ tiles, int B, int T, int Tk, int H,
                                             long long tile_stride, long long idx, const int* key_lens) {   // idx = (bh, key8, d)
  const long long total = (long long)B * H * (Tk / 8) * 128;
  if (idx >= total) return;
  const int d = (int)(idx % 128);
  const long long r = idx / 128;
  const int k8 = (int)(r % (Tk / 8));
  const int bh = (int)(r / (Tk / 8));
  const int b = bh / H, h = bh - b * H;
  const int D = H * 128;
  const int rows = af_key_rows<RAG>(key_lens, T, b);
  if (RAG && k8 * 8 >= (rows + 127) / 128 * 128) return;
  float f[8];
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const int key = k8 * 8 + e;
    f[e] = key < rows ? __ldg(qkv + ((long long)b * T + key) * 3 * D + 2 * D + h * 128 + d) : 0.f;
  }
  uint4 hi, lo;
  split8(f, AF_WSCALE, hi, lo);
  unsigned char* base = tiles + (long long)bh * tile_stride;
  if (k8 == 0 && d == 0) *reinterpret_cast<float*>(base) = 1.f / AF_WSCALE;
  const int kb = k8 >> 1, chunk = k8 & 1;
  const size_t b_plane = AF_STAGE / 2;
  unsigned char* dst = base + TC_HDR + (size_t)kb * AF_STAGE + ((size_t)chunk * 128 + d) * 16;
  *reinterpret_cast<uint4*>(dst) = hi;
  *reinterpret_cast<uint4*>(dst + b_plane) = lo;
}

// One launch writes both operand-tile sets: blocks [0, k_blocks) the K tiles, the rest the V tiles.
template <bool RAG>
__global__ void pack_kv_tiles_kernel(const float* __restrict__ qkv, unsigned char* __restrict__ kt, unsigned char* __restrict__ vt, int B, int T,
                                     int Tk, int H, long long tile_stride, unsigned k_blocks, const int* key_lens) {
  if (blockIdx.x < k_blocks) pack_k_tiles<RAG>(qkv, kt, B, T, Tk, H, tile_stride, (long long)blockIdx.x * blockDim.x + threadIdx.x, key_lens);
  else pack_v_tiles<RAG>(qkv, vt, B, T, Tk, H, tile_stride, (long long)(blockIdx.x - k_blocks) * blockDim.x + threadIdx.x, key_lens);
}

// ------------------------------------------------------------------ attention kernel

struct AfP {
  const float* qkv; float* ctx;
  const unsigned char* kt; const unsigned char* vt; long long tstride;     // per (b, h) tile buffers (128-byte header first)
  int B, T, H;
  const int* key_lens; float scale;
  int qtiles, n_items;                           // work items of the padded shape: per (utterance, head), in all
};

// 16 fp32 values of one row -> fp16 hi / lo operand planes of K-block kb ([2 chunks][128 rows][16 B] each)
__device__ __forceinline__ void af_store16(unsigned char* kblk, int row, const float (&a)[16]) {
  uint32_t hw[8], lw[8];
#pragma unroll
  for (int j = 0; j < 8; j++) hw[j] = split_f16x2(a[2 * j], a[2 * j + 1], lw[j]);
  unsigned char* p0 = kblk + (size_t)row * 16;
  *reinterpret_cast<uint4*>(p0) = make_uint4(hw[0], hw[1], hw[2], hw[3]);                 // hi, chunk 0
  *reinterpret_cast<uint4*>(p0 + 2048) = make_uint4(hw[4], hw[5], hw[6], hw[7]);          // hi, chunk 1
  *reinterpret_cast<uint4*>(p0 + 4096) = make_uint4(lw[0], lw[1], lw[2], lw[3]);          // lo, chunk 0
  *reinterpret_cast<uint4*>(p0 + 6144) = make_uint4(lw[4], lw[5], lw[6], lw[7]);          // lo, chunk 1
}

__device__ __forceinline__ void af_wg_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(g + 1) : "memory"); }   // one warpgroup

template <bool RAG>
__global__ void __launch_bounds__(AF_THREADS, 1) attention_fused_kernel(const AfP p) {
  constexpr uint32_t KBLK = 8192;                // one 16-wide K-block of an A operand: hi plane 4 KB + lo plane 4 KB (128 rows)
  constexpr uint32_t PLANES = 8 * KBLK;          // 128 x 128 operand: 64 KB
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int tid = threadIdx.x, warp = warp_uniform_id(), lane = tid & 31;
  unsigned char* qa = smem_raw;                  // Q operand planes
  unsigned char* pa = qa + PLANES;               // P operand planes
  unsigned char* ring = pa + PLANES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + (size_t)AF_SB * AF_STAGE);
  uint64_t* fullB = bars;                        // [AF_SB]
  uint64_t* emptyB = fullB + AF_SB;              // [AF_SB]

  if (tid == 0) {
    ring_init(fullB, emptyB, AF_SB, 1, 8);
    mbar_init_fence();
  }
  __syncthreads();
  // Items are (head, utterance, query tile), heads as the block dimension; each streams the key blocks of its utterance's rows.
  WorkList<RAG, AF_MIN_ROWS> work;
  work.init(p.key_lens, 1, p.T, p.B, 128, p.qtiles, p.n_items);

  if (warp == 8) {
    // ===================== K / V stage producer, in the order the consumers read them =====================
    if (lane == 0) {
      Ring rb;
      auto push = [&](const unsigned char* src) { ring_push(fullB, emptyB, rb, AF_SB, ring + (size_t)rb.idx * AF_STAGE, src, AF_STAGE); };
      for (int item = blockIdx.x; item < work.count; item += gridDim.x) {
        const Item it = work.item(item);
        const int bh = it.b * p.H + it.nblk, nkb_i = (it.rows + 127) / 128;
        const unsigned char* kt = p.kt + (long long)bh * p.tstride + TC_HDR;   // [key block][d/16][8 KB]
        const unsigned char* vt = p.vt + (long long)bh * p.tstride + TC_HDR;   // [key/16][8 KB]
        for (int j = 0; j < nkb_i; j++)                                          // pass 1
          for (int kb = 0; kb < 8; kb++) push(kt + ((size_t)j * 8 + kb) * AF_STAGE);
        for (int j = 0; j < nkb_i; j++) {                                        // pass 2
          for (int kb = 0; kb < 8; kb++) push(kt + ((size_t)j * 8 + kb) * AF_STAGE);   // S(j)
          for (int kb = 0; kb < 8; kb++) push(vt + ((size_t)j * 8 + kb) * AF_STAGE);   // P V_j
        }
      }
    }
    return;
  }
  // ===================== consumer warpgroups =====================
  const int g = warp >> 2, w = warp & 3;
  const int D = p.H * 128;
  const float c = p.scale * (1.f / AF_WSCALE) * 1.4426950408889634f;      // s*c = scaled score in log2 units (K tiles carry x16)
  const uint64_t desc_c = wgmma_desc(0, 2048, 128);    // A and B alike: chunk stride 128 rows * 16 B, 8-row groups 128 B apart
  const uint32_t qa16 = (smem_u32(qa) >> 4) + 64 * g, pa16 = (smem_u32(pa) >> 4) + 64 * g;
  Ring rb;
  // D (+)= A(planes a16, 8 K-blocks) x B(next 8 ring stages), three-MMA split.  acc0 = 0: the first MMA overwrites D.
  auto gemm = [&](uint32_t a16, float (&d)[64], uint32_t acc0) {
    int pend = -1;
    for (int kb = 0; kb < 8; kb++, rb.advance(AF_SB))
      ring_step(fullB, emptyB, rb, pend, [&](uint32_t sb) {
        const uint64_t a_hi = desc_c | (uint64_t)((a16 + kb * (KBLK >> 4)) & 0x3fff), a_lo = a_hi + (4096 >> 4);
        const uint64_t b_hi = desc_c | (uint64_t)(smem_u32(ring + (size_t)sb * AF_STAGE) >> 4), b_lo = b_hi + (4096 >> 4);
        Wgmma<128>::f16(d, a_lo, b_hi, kb == 0 ? acc0 : 1u);
        Wgmma<128>::f16(d, a_hi, b_hi, 1u);
        Wgmma<128>::f16(d, a_hi, b_lo, 1u);
      });
    ring_drain(emptyB, pend);
    wgmma_keep<128>(d);
  };
  const int qr = (tid & 127) >> 1, qhalf = tid & 1;    // Q conversion: row, 64-column half
  for (int item = blockIdx.x; item < work.count; item += gridDim.x) {
    const Item it = work.item(item);
    const int b = it.b, hd = it.nblk, rows = it.rows, nkb_i = (rows + 127) / 128;   // rows that exist: the utterance's own in ragged mode
    const int len = p.key_lens ? min(p.key_lens[b], p.T) : p.T;                      // keys >= len are masked (ragged: len = rows)
    // ---- Q rows of this warpgroup -> operand planes (the previous item's MMAs have all retired)
    {
      const int t = it.t0 + 64 * g + qr;
      const float* src = p.qkv + ((long long)b * p.T + t) * 3 * D + hd * 128 + qhalf * 64;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        float v[16];
        if (t < rows) {
#pragma unroll
          for (int k4 = 0; k4 < 4; k4++) {
            const float4 u = __ldg(reinterpret_cast<const float4*>(src + k * 16) + k4);
            v[4 * k4] = u.x; v[4 * k4 + 1] = u.y; v[4 * k4 + 2] = u.z; v[4 * k4 + 3] = u.w;
          }
        } else {
#pragma unroll
          for (int i = 0; i < 16; i++) v[i] = 0.f;
        }
        af_store16(qa + (size_t)(qhalf * 4 + k) * KBLK, 64 * g + qr, v);
      }
      fence_proxy_async();
      af_wg_sync(g);
    }
    float sacc[64];
    // ---- pass 1: row maxima of the masked, scaled scores (rows lane/4 and lane/4 + 8 of this warp's 16)
    float m[2] = {-INFINITY, -INFINITY};
    for (int j = 0; j < nkb_i; j++) {
      gemm(qa16, sacc, 0u);
#pragma unroll
      for (int jj = 0; jj < 16; jj++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const int key = j * 128 + 8 * jj + 2 * (lane & 3) + e;
          if (key < len) {
            m[0] = fmaxf(m[0], sacc[4 * jj + e] * c);
            m[1] = fmaxf(m[1], sacc[4 * jj + 2 + e] * c);
          }
        }
    }
#pragma unroll
    for (int h = 0; h < 2; h++) {
      m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 1));
      m[h] = fmaxf(m[h], __shfl_xor_sync(0xffffffffu, m[h], 2));
    }
    // ---- pass 2: p = exp2(s*c - m) x AF_PSCALE -> P operand planes -> O += P V_j.  The scale is applied after exp2f, so that p itself
    // rounds as it would unscaled; l carries it too, so O / l needs no correction.
    float oacc[64];
    float l[2] = {0.f, 0.f};
    const int prow = 64 * g + 16 * w + (lane >> 2);
    for (int j = 0; j < nkb_i; j++) {
      gemm(qa16, sacc, 0u);
#pragma unroll
      for (int jj = 0; jj < 16; jj++) {
        const int k0 = 8 * jj + 2 * (lane & 3);          // key inside the block
        unsigned char* base = pa + (size_t)(k0 >> 4) * KBLK + ((k0 >> 3) & 1) * 2048 + (k0 & 7) * 2;
#pragma unroll
        for (int h = 0; h < 2; h++) {
          float e[2];
#pragma unroll
          for (int q = 0; q < 2; q++) {
            e[q] = j * 128 + k0 + q < len ? exp2f(fmaf(sacc[4 * jj + 2 * h + q], c, -m[h])) * AF_PSCALE : 0.f;
            l[h] += e[q];
          }
          uint32_t lw;
          const uint32_t hw = split_f16x2(e[0], e[1], lw);
          unsigned char* rowp = base + (size_t)(prow + 8 * h) * 16;
          *reinterpret_cast<uint32_t*>(rowp) = hw;
          *reinterpret_cast<uint32_t*>(rowp + 4096) = lw;
        }
      }
      fence_proxy_async();
      af_wg_sync(g);                                   // every thread's P values are in place before the warpgroup's MMAs read them
      if (j == 0) {
#pragma unroll
        for (int i = 0; i < 64; i++) oacc[i] = 0.f;
      }
      gemm(pa16, oacc, 1u);                            // O += P V_j (zeroed above for the first key block)
      af_wg_sync(g);                                   // the P planes are rewritten by the next key block
    }
    // ---- epilogue: O / l (V tiles carry x16), rows beyond the utterance are zero
#pragma unroll
    for (int h = 0; h < 2; h++) {
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
      l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
      const int t = it.t0 + prow + 8 * h;
      if (t >= rows) continue;
      const float inv = t < len ? (1.f / AF_WSCALE) / l[h] : 0.f;
      float* dst = p.ctx + ((long long)b * p.T + t) * D + hd * 128 + 2 * (lane & 3);
#pragma unroll
      for (int jj = 0; jj < 16; jj++)
        *reinterpret_cast<float2*>(dst + 8 * jj) = make_float2(oacc[4 * jj + 2 * h] * inv, oacc[4 * jj + 2 * h + 1] * inv);
    }
  }
}

static constexpr size_t AF_SMEM = 2 * 65536 + (size_t)AF_SB * AF_STAGE + 2 * AF_SB * 8 + 16;

static inline long long af_tile_stride(int Tk) { return TC_HDR + (long long)Tk * 512; }

size_t attention_fused_workspace(int B, int T, int H) {
  const int Tk = (T + 127) / 128 * 128;
  const size_t tile_bytes = ((size_t)B * H * af_tile_stride(Tk) + 255) & ~(size_t)255;
  return 2 * tile_bytes + 256;
}

int attention_fused(const fs2_attention_args* a, void* ws, size_t ws_bytes, cudaStream_t s, bool ragged) {
  if (!a || !a->qkv || !a->ctx || !ws || a->B <= 0 || a->T <= 0 || a->H <= 0) return FS2_ERR_ARG;
  if (a->Dh != 128) return FS2_ERR_UNSUPPORTED;
  if (!aligned16(a->qkv) || !aligned16(a->ctx)) return FS2_ERR_ARG;
  if (ws_bytes < attention_fused_workspace(a->B, a->T, a->H)) return FS2_ERR_WORKSPACE;
  int derr = FS2_OK;
  DevState* dv = dev_state(&derr);
  if (!dv) return derr;
  if (ragged && !a->key_lens) return FS2_ERR_ARG;
  FS2_TRY(dev_once(dv->att_fused_ready, [] {
    const cudaError_t e = cudaFuncSetAttribute(attention_fused_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AF_SMEM);
    return e == cudaSuccess ? cudaFuncSetAttribute(attention_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)AF_SMEM) : e;
  }));
  const int Tk = (a->T + 127) / 128 * 128;
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 255) & ~(uintptr_t)255);
  const long long tstride = af_tile_stride(Tk);
  const size_t tile_bytes = ((size_t)a->B * a->H * tstride + 255) & ~(size_t)255;
  unsigned char* kt = reinterpret_cast<unsigned char*>(base);
  unsigned char* vt = kt + tile_bytes;
  {
    const long long nk = (long long)a->B * a->H * Tk * (128 / 8), nv = (long long)a->B * a->H * (Tk / 8) * 128;
    const unsigned kb = (unsigned)((nk + 255) / 256), vb = (unsigned)((nv + 255) / 256);
    prof_before(s);
    if (ragged) pack_kv_tiles_kernel<true><<<kb + vb, 256, 0, s>>>(a->qkv, kt, vt, a->B, a->T, Tk, a->H, tstride, kb, a->key_lens);
    else pack_kv_tiles_kernel<false><<<kb + vb, 256, 0, s>>>(a->qkv, kt, vt, a->B, a->T, Tk, a->H, tstride, kb, nullptr);
    prof_after(s, 1, 0.0);
    FS2_LAUNCH_CHECK();
  }
  AfP p{};
  p.qkv = a->qkv; p.ctx = a->ctx; p.kt = kt; p.vt = vt; p.tstride = tstride;
  p.B = a->B; p.T = a->T; p.H = a->H; p.key_lens = a->key_lens; p.scale = a->scale;
  p.qtiles = Tk / 128;
  const long long items = (long long)a->B * a->H * p.qtiles;
  if (items > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
  p.n_items = (int)items;
  const int num_sms = dv->num_sms.load(std::memory_order_relaxed);
  const int grid = items < num_sms ? (int)items : num_sms;
  prof_before(s);
  if (ragged) attention_fused_kernel<true><<<grid, AF_THREADS, AF_SMEM, s>>>(p);   // grid from the padded shape: CTAs without work exit
  else attention_fused_kernel<false><<<grid, AF_THREADS, AF_SMEM, s>>>(p);
  // algorithmic count as the reference computes it (dense T x T): 4*T*T*Dh per (b, h)
  prof_after(s, 1, 4.0 * a->B * a->H * (double)a->T * a->T * 128);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
