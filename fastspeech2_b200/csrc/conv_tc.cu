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

// K-segmented evaluation in ONE launch (FS2_TC_VARIANT_SEGMENTED): the work units are (tile, tap, 256-channel chunk) slices, and the
// plan is made for the shape of one slice (`slice`: Cin = 256, one tap).  Other variants: nseg = 1 and the plan is made for `a` itself.
// Returns the arguments to plan on, or NULL if the segmented variant cannot take the shape.
static const fs2_conv1d_args* conv_tc_segments(const fs2_conv1d_args* a, fs2_conv1d_args& slice, int& nseg, int& seg_nkc) {
  nseg = seg_nkc = 1;
  if (!(a->tc_variant & FS2_TC_VARIANT_SEGMENTED)) return a;
  if (!(a->tc_variant & FS2_TC_VARIANT_NB64) || a->Cin % 256 || a->N % 64 || a->dilation != 1 || a->alpha != 1.f || a->out_act != FS2_ACT_NONE)
    return nullptr;
  seg_nkc = a->Cin / 256; nseg = a->taps * seg_nkc;
  slice = *a;
  slice.Cin = 256; slice.taps = 1;
  return &slice;
}

// Shape-derived launch plan (pure host logic, no CUDA calls): work-item shape, accumulator grouping, ring depths, shared-memory
// budget, grid.  nseg: K-segments per tile (conv_tc_segments).  Returns FS2_OK or FS2_ERR_UNSUPPORTED.  Exposed as fs2_conv_tc_plan so
// that the heuristics' invariants are testable without a GPU (tests/test_abi.py).
static int conv_tc_plan(const fs2_conv1d_args* a, int nseg, int num_sms, fs2_conv_tc_plan_t& p) {
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
  p.acc_regs = p.TG * p.NB / 2;
  // ring barriers, and the staged epilogue tiles of a conv with a residual, accumulate or K-segments (conv_tc_kernel.cuh)
  const size_t fixed = TC_RING_BAR_BYTES + tc_stage_bytes(p.NB, tc_stage_tiles(a->res != nullptr, a->accumulate != 0, nseg));
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
  p.tiles_per_batch = (a->T + 127) / 128;
  const long long n_items = (long long)(a->N / p.NB) * a->B * p.tiles_per_batch;
  if (n_items > 0x7fffffffLL) return FS2_ERR_UNSUPPORTED;
  p.n_items = (int)n_items;
  // Channel-block groups: a work item computes NG blocks from one resident slab (all kblocks stages), so the transform warps load and
  // split each input tile once instead of N / NB times, and read it from HBM once.  The largest NG that fits the budget with a weight ring
  // of >= 2 stages, keeps >= 4 waves of items (the tail wave's idle SMs stay <= 1/4 of the launch) and divides the blocks.
  p.NG = 1;
  const int nblocks = a->N / p.NB;
  if (nseg == 1 && kblocks <= TC_SA_MAX)
    for (int ng = nblocks; ng > 1 && p.NG == 1; ng--) {
      if (nblocks % ng || n_items / ng < 4LL * num_sms) continue;
      int gsa = TC_SA_MAX, gsb = sb;
      while (fixed + gsa * a_stage + gsb * b_stage > budget && gsa > kblocks) gsa--;
      while (fixed + gsa * a_stage + gsb * b_stage > budget && gsb > 2) gsb--;
      if (fixed + gsa * a_stage + gsb * b_stage > budget) continue;
      p.NG = ng; sa = gsa; sb = gsb;
    }
  p.SA = sa; p.SB = sb;
  p.smem = (int)(fixed + sa * a_stage + sb * b_stage);   // [slab stages][weight stages][ring barriers][staged inputs]
  const long long ctas = n_items / p.NG;
  p.grid = ctas < num_sms ? (int)ctas : num_sms;
  return FS2_OK;
}

int conv_tc_plan_query(const fs2_conv1d_args* a, int num_sms, fs2_conv_tc_plan_t* out) {
  if (!a || !out || num_sms <= 0 || a->B <= 0 || a->T <= 0 || a->Cin <= 0 || a->N <= 0 || a->taps <= 0) return FS2_ERR_ARG;
  if (!conv_tc_supported(a)) return FS2_ERR_UNSUPPORTED;
  fs2_conv1d_args slice;
  int nseg, seg_nkc;
  const fs2_conv1d_args* plan_args = conv_tc_segments(a, slice, nseg, seg_nkc);
  if (!plan_args) return FS2_ERR_UNSUPPORTED;
  fs2_conv_tc_plan_t pl{};
  const int rc = conv_tc_plan(plan_args, nseg, num_sms, pl);
  if (rc == FS2_OK) *out = pl;
  return rc;
}

// a->w_tc must be the tiled layout produced by fastspeech2_b200.packing.pack_conv_tc (see fs2b200.h) in the format a->tc_variant names.
// win (with a->x_lens): NULL, or the windowed mode (OriginWindow; a->T is not used): the plan is made for the window's rows.
// lw: NULL, or the table mode (LaunchWeights): a->w_tc and a->bias are model 0's, every work item reads its utterance's model's.
int conv1d_tc(const fs2_conv1d_args* a, cudaStream_t s, const OriginWindow* win, const LaunchWeights* lw) {
  if (!a || !a->x || !a->w_tc || !a->y) return FS2_ERR_ARG;
  if (a->B <= 0 || a->T <= 0 || a->Cin <= 0 || a->N <= 0 || a->taps <= 0) return FS2_ERR_ARG;
  if (!conv_tc_supported(a)) return FS2_ERR_UNSUPPORTED;
  if (!aligned16(a->x) || !aligned16(a->w_tc) || !aligned16(a->y) || (a->res && !aligned16(a->res))) return FS2_ERR_ARG;
  if (win && !a->x_lens) return FS2_ERR_ARG;
  const unsigned variant = a->tc_variant;
  fs2_conv1d_args slice, rows;
  int nseg, seg_nkc;
  const fs2_conv1d_args* plan_args = conv_tc_segments(a, slice, nseg, seg_nkc);
  if (!plan_args) return FS2_ERR_UNSUPPORTED;
  if (win) {                                            // tiles of the window only
    if (win->rows.yend <= win->rows.y0) return FS2_ERR_ARG;
    rows = *plan_args;
    rows.T = win->rows.yend - win->rows.y0;
    plan_args = &rows;
  }
  int derr = FS2_OK;
  DevState* dv = dev_state(&derr);                      // state of the CURRENT device: the caller's stream must belong to it
  if (!dv) return derr;
  FS2_TRY(dev_once(dv->conv_tc_ready, [] {
    const int mx = 227 * 1024;
    cudaError_t e = cudaSuccess;
    for (cudaError_t (*prep)(int) : {conv_tc_prepare_nb16, conv_tc_prepare_nb32, conv_tc_prepare_nb48, conv_tc_prepare_nb64,
                                     conv_tc_prepare_nb80, conv_tc_prepare_nb96, conv_tc_prepare_nb112, conv_tc_prepare_nb128})
      if (e == cudaSuccess) e = prep(mx);
    return e;
  }));
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
  fs2_conv_tc_plan_t pl{};
  FS2_TRY(conv_tc_plan(plan_args, nseg, g_num_sms, pl));
  p.SA = pl.SA; p.SB = pl.SB; p.TPS = pl.TPS; p.R = pl.R; p.tiles_per_batch = pl.tiles_per_batch;
  p.NG = pl.NG; p.n_items = pl.n_items / pl.NG;         // the kernel's items: tiles x groups of NG channel blocks
  p.stage_off = pl.smem - (int)tc_stage_bytes(pl.NB, tc_stage_tiles(a->res != nullptr, a->accumulate != 0, nseg));   // the staged inputs end the budget
  p.win = win ? win->rows : RowWindow{0, a->T, a->T};
  p.org = win ? win->org : nullptr;
  static_assert(226 * 1024 + TC_TABLE_SLOT_BYTES <= 227 * 1024, "the slot ring fits between the plan's budget and the opt-in");
  p.slot_off = pl.smem;                                 // the unit slot ring (TcSlot) follows the plan's budget, within the 227 KB opt-in
  const size_t smem = (size_t)pl.smem + (lw ? TC_TABLE_SLOT_BYTES : TC_SLOT_BYTES);
  if (lw) { p.table = lw->t; p.wt_ref = lw->wt; p.bias_ref = lw->bias; }
  const unsigned grid = (unsigned)pl.grid;
  const bool w = win != nullptr;
  prof_before(s);
  switch (pl.NB) {
    case 16: conv_tc_launch_nb16(p, w, grid, smem, s); break;
    case 32: conv_tc_launch_nb32(p, w, grid, smem, s); break;
    case 48: conv_tc_launch_nb48(p, w, grid, smem, s); break;
    case 64: conv_tc_launch_nb64(p, w, grid, smem, s); break;
    case 80: conv_tc_launch_nb80(p, w, grid, smem, s); break;
    case 96: conv_tc_launch_nb96(p, w, grid, smem, s); break;
    case 112: conv_tc_launch_nb112(p, w, grid, smem, s); break;
    default: conv_tc_launch_nb128(p, w, grid, smem, s); break;
  }
  prof_after(s, 0, 2.0 * a->B * plan_args->T * (double)a->Cin * a->taps * a->N);
  FS2_LAUNCH_CHECK();
  return FS2_OK;
}

}  // namespace fs2
