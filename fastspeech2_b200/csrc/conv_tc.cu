// Host side of the wgmma implicit-GEMM Conv1d: shape support, work-item / ring heuristics, launch.
// Device code: conv_tc_kernel.cuh (instantiated in conv_tc_nb*.cu).
#include "conv_tc_kernel.cuh"

namespace fs2 {

// ------------------------------------------------------------------ host side
// Output channels per work item: NB <= 128 keeps a consumer thread's accumulators at <= 64 registers.  The f8 split asks for
// nb_max = 64: Hopper accumulates E4M3 products with reduced precision, so its correction term needs an accumulator of its own.
int conv_tc_nb(int N, int nb_max) {
  if (N % 16) return 0;
  if (N <= nb_max) return N;
  for (int nb = nb_max; nb >= 16; nb -= 16)
    if (N % nb == 0) return nb;
  return 0;
}

bool conv_tc_supported(const fs2_conv1d_args* a) {
  if (!a || a->Cin % TC_KB || a->N % 16 || conv_tc_nb(a->N, 128) == 0) return false;
  if ((a->x_row_stride & 7) || (a->x_batch_stride & 7) || (reinterpret_cast<uintptr_t>(a->x) & 31u)) return false;   // 256-bit loads
  if ((a->y_row_stride & 3) || (a->y_batch_stride & 3)) return false;
  if ((long long)(TC_LD * TC_TTHREADS) * a->x_row_stride > 0x7fffffffLL) return false;                                // 32-bit row offsets
  if (a->res && ((a->res_row_stride & 3) || (a->res_batch_stride & 3))) return false;
  if (a->in_act != FS2_ACT_NONE && a->in_act != FS2_ACT_LRELU) return false;
  if (a->in_act == FS2_ACT_LRELU && !(a->in_slope >= 0.f && a->in_slope <= 1.f)) return false;   // max(x, slope*x) form
  if ((a->taps - 1) * a->dilation > TC_LD * TC_TTHREADS / TC_CHUNKS - 128) return false;   // slab rows the transform warps hold
  return true;
}

// Shape-derived launch plan (pure host logic, no CUDA calls): work-item shape, accumulator grouping, ring depths, shared-memory
// budget, grid.  Returns FS2_OK or FS2_ERR_UNSUPPORTED.  Exposed as fs2_conv_tc_plan so that the heuristics' invariants are
// testable without a GPU (tests/test_abi.py).
static int conv_tc_plan(const fs2_conv1d_args* a, int num_sms, TcP& p, size_t& smem, int& grid) {
  const bool nb64 = (a->tc_variant & FS2_TC_VARIANT_NB64) != 0;   // 64-channel work items: separate accumulators for hi*hi and the cross terms
  const bool f8 = (a->tc_variant & FS2_TC_VARIANT_F8) != 0;
  p.NB = nb64 ? (a->N % 64 == 0 ? 64 : (a->N < 64 && a->N % 16 == 0 ? a->N : 0)) : conv_tc_nb(a->N, f8 ? 64 : 128);
  if (p.NB == 0) return FS2_ERR_UNSUPPORTED;
  const int halo = (a->taps - 1) * a->dilation;
  // One 128-row tile per work item, split between the two consumer warpgroups.  Narrow blocks (NB <= 64): hi*hi and the two cross
  // terms accumulate in separate register sets (summed in fp32 round-to-nearest by the epilogue) at the same register cost as NB = 128.
  int R = 128 + halo;
  R += (12 - (R & 7)) & 7;                             // R % 8 == 4: conflict-free transform stores (2 chunks per row)
  if (R > TC_LD * TC_TTHREADS / TC_CHUNKS + 7) return FS2_ERR_UNSUPPORTED;
  p.R = R;
  p.TG = p.NB <= 64 ? 2 : 1;
  const size_t fixed = (2 * TC_SA_MAX + 2 * TC_SB_MAX) * 8 + 16;
  const size_t tap_bytes = (size_t)2 * TC_CHUNKS * p.NB * 16;
  int tps = a->taps >= 5 ? 4 : 1;                      // taps per weight stage: wide kernels share one bulk copy / handshake
  if (tps > a->taps) tps = a->taps;
  p.TPS = tps;
  const size_t a_stage = (size_t)2 * TC_CHUNKS * R * 16, b_stage = (size_t)tps * tap_bytes;
  const size_t budget = 226 * 1024;
  const int kblocks = a->Cin / TC_KB;
  // Slab ring depth: the ring spans work items, so even 2-K-block layers want 3 stages; short kernels have the least MMA work per
  // slab and the deepest ring.
  int sa = 3, sb = tps > 1 ? 4 : TC_SB_MAX;
  if (a->taps <= 3) sa = 5;
  else if (kblocks >= 4) sa = 4;
  while (fixed + sa * a_stage + sb * b_stage > budget && sa > 3) sa--;
  while (fixed + sa * a_stage + sb * b_stage > budget && sb > 3) sb--;
  while (fixed + sa * a_stage + sb * b_stage > budget && sa > 2) sa--;
  while (fixed + sa * a_stage + sb * b_stage > budget && sb > 2) sb--;
  if (fixed + sa * a_stage + sb * b_stage > budget) return FS2_ERR_UNSUPPORTED;
  p.SA = sa; p.SB = sb;
  smem = fixed + sa * a_stage + sb * b_stage;
  p.tiles_per_batch = (a->T + 127) / 128;
  const long long n_items = (long long)(a->N / p.NB) * a->B * p.tiles_per_batch;
  if (n_items > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
  p.n_items = (int)n_items;
  grid = n_items < num_sms ? (int)n_items : num_sms;
  return FS2_OK;
}

// out[11] = {NB, TG, SA, SB, TPS, R, accumulator registers per consumer thread, tiles_per_batch, n_items, grid, dynamic smem bytes}
int conv_tc_plan_query(const fs2_conv1d_args* a, int num_sms, int* out) {
  if (!a || !out || num_sms <= 0 || a->B <= 0 || a->T <= 0 || a->Cin <= 0 || a->N <= 0 || a->taps <= 0) return FS2_ERR_ARG;
  if (!conv_tc_supported(a)) return FS2_ERR_UNSUPPORTED;
  TcP p{};
  size_t smem = 0;
  int grid = 0;
  const int rc = conv_tc_plan(a, num_sms, p, smem, grid);
  if (rc != FS2_OK) return rc;
  const int v[11] = {p.NB, p.TG, p.SA, p.SB, p.TPS, p.R, p.TG * p.NB / 2, p.tiles_per_batch, p.n_items, grid, (int)smem};
  for (int i = 0; i < 11; i++) out[i] = v[i];
  return FS2_OK;
}

// a->w_tc must be the tiled layout produced by fastspeech2_b200.packing.pack_conv_tc (see fs2b200.h) in the format a->tc_variant names
int conv1d_tc(const fs2_conv1d_args* a, cudaStream_t s) {
  if (!a || !a->x || !a->w_tc || !a->y) return FS2_ERR_ARG;
  if (a->B <= 0 || a->T <= 0 || a->Cin <= 0 || a->N <= 0 || a->taps <= 0) return FS2_ERR_ARG;
  if (!conv_tc_supported(a)) return FS2_ERR_UNSUPPORTED;
  if (!aligned16(a->x) || !aligned16(a->w_tc) || !aligned16(a->y) || (a->res && !aligned16(a->res))) return FS2_ERR_ARG;
  const unsigned variant = a->tc_variant;
  // K-segmented evaluation in ONE launch (FS2_TC_VARIANT_SEGMENTED): the work units are (tile, tap, 256-channel chunk)
  fs2_conv1d_args seg_args;
  int nseg = 1, seg_nkc = 1;
  if (variant & FS2_TC_VARIANT_SEGMENTED) {
    if (!(variant & FS2_TC_VARIANT_NB64) || a->Cin % 256 || a->N % 64 || a->dilation != 1 || a->alpha != 1.f || a->out_act != FS2_ACT_NONE)
      return FS2_ERR_UNSUPPORTED;
    seg_nkc = a->Cin / 256; nseg = a->taps * seg_nkc;
    seg_args = *a;
    seg_args.Cin = 256; seg_args.taps = 1;          // shape of one slice: ring / tile planning happens on this
  }
  const fs2_conv1d_args* plan_args = nseg > 1 || (variant & FS2_TC_VARIANT_SEGMENTED) ? &seg_args : a;
  int derr = FS2_OK;
  DevState* dv = dev_state(&derr);                      // state of the CURRENT device: the caller's stream must belong to it
  if (!dv) return derr;
  if (!dv->conv_tc_ready.load(std::memory_order_acquire)) {
    DevOnce once;
    if (!dv->conv_tc_ready.load(std::memory_order_relaxed)) {
      const int mx = 227 * 1024;
      cudaError_t e = cudaSuccess;
      for (cudaError_t (*prep)(int) : {conv_tc_prepare_nb16, conv_tc_prepare_nb32, conv_tc_prepare_nb48, conv_tc_prepare_nb64,
                                       conv_tc_prepare_nb80, conv_tc_prepare_nb96, conv_tc_prepare_nb112, conv_tc_prepare_nb128})
        if (e == cudaSuccess) e = prep(mx);
      if (e != cudaSuccess) return FS2_ERR_CUDA - (int)e;
      dv->conv_tc_ready.store(true, std::memory_order_release);
    }
  }
  const int g_num_sms = dv->num_sms.load(std::memory_order_relaxed);
  TcP p{};
  p.x = a->x; p.xbs = a->x_batch_stride; p.xrs = a->x_row_stride;
  p.B = a->B; p.T = a->T; p.Cin = plan_args->Cin;
  p.wt = a->w_tc; p.bias = a->bias; p.N = a->N;
  p.taps = plan_args->taps; p.dil = a->dilation; p.pad = a->pad_left;
  p.nseg = nseg; p.seg_nkc = seg_nkc; p.seg_wbytes = TC_HDR + (long long)1024 * a->N;
  p.in_act = a->in_act; p.in_slope = a->in_slope; p.out_act = a->out_act; p.out_slope = a->out_slope;
  p.res = a->res; p.rbs = a->res_batch_stride; p.rrs = a->res_row_stride;
  p.alpha = a->alpha; p.accumulate = a->accumulate; p.row_lens = a->row_lens;
  p.y = a->y; p.ybs = a->y_batch_stride; p.yrs = a->y_row_stride;
  p.f8 = (variant & FS2_TC_VARIANT_F8) ? 1 : 0;
  p.x_lens = a->x_lens; p.lens_scale = a->lens_scale;   // the plan below stays the padded one: the host never reads device lengths
  size_t smem = 0;
  int grid = 0;
  const int rc = conv_tc_plan(plan_args, g_num_sms, p, smem, grid);
  if (rc != FS2_OK) return rc;
  prof_before(s);
  switch (p.NB) {
    case 16: conv_tc_launch_nb16(p, (unsigned)grid, smem, s); break;
    case 32: conv_tc_launch_nb32(p, (unsigned)grid, smem, s); break;
    case 48: conv_tc_launch_nb48(p, (unsigned)grid, smem, s); break;
    case 64: conv_tc_launch_nb64(p, (unsigned)grid, smem, s); break;
    case 80: conv_tc_launch_nb80(p, (unsigned)grid, smem, s); break;
    case 96: conv_tc_launch_nb96(p, (unsigned)grid, smem, s); break;
    case 112: conv_tc_launch_nb112(p, (unsigned)grid, smem, s); break;
    default: conv_tc_launch_nb128(p, (unsigned)grid, smem, s); break;
  }
  prof_after(s, 0, 2.0 * a->B * a->T * (double)a->Cin * a->taps * a->N);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
