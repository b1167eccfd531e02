// Host side of the fused SS2D scan: tensor maps, L-segment planning, dispatch (sigma_ss2d_scan_fwd).
#include <stdlib.h>

#include <algorithm>
#include <string>

#include "ss2d_scan.cuh"

namespace sigma {

// ---- tensor maps: the one caller of cuTensorMapEncodeTiled, through the runtime-resolved driver entry point ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void *ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
    set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  fn = (EncodeTiledFn)ptr;
  return fn;
}

int make_tmap(CUtensorMap *map, CUtensorMapDataType dtype, int rank, const void *base, const uint64_t *dims,
              const uint64_t *strides_bytes, const uint32_t *box, CUtensorMapSwizzle swz, CUtensorMapL2promotion promo) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return SIGMA_ECUDA;
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bdim[i] = box[i]; estr[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(map, dtype, (cuuint32_t)rank, const_cast<void *>(base), gdim, gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                  promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    std::string d, st, bx;
    for (int i = 0; i < rank; ++i) {
      d += (i ? "," : "") + std::to_string(dims[i]);
      bx += (i ? "," : "") + std::to_string(box[i]);
      if (i + 1 < rank) st += (i ? "," : "") + std::to_string(strides_bytes[i]);
    }
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): rank=%d dims=(%s) strides=(%s) box=(%s) base=%p", (int)r, rank, d.c_str(),
              st.c_str(), bx.c_str(), base);
    return SIGMA_ECUDA;
  }
  return SIGMA_OK;
}

int pad_rp(int R) {
  const int opts[] = {4, 8, 12, 16, 24, 32, 48, 64};
  for (int o : opts)
    if (R <= o) return o;
  return -1;
}

template <int N, int CPT>
static int dispatch_rp(const Ss2dParams &p, int nthreads, int ctas, cudaStream_t s) {
  switch (pad_rp(p.R)) {
    case 4: return ss2d_launch<N, CPT, 4>(p, nthreads, ctas, s);
    case 8: return ss2d_launch<N, CPT, 8>(p, nthreads, ctas, s);
    case 12: return ss2d_launch<N, CPT, 12>(p, nthreads, ctas, s);
    case 16: return ss2d_launch<N, CPT, 16>(p, nthreads, ctas, s);
    case 24: return ss2d_launch<N, CPT, 24>(p, nthreads, ctas, s);
    case 32: return ss2d_launch<N, CPT, 32>(p, nthreads, ctas, s);
    case 48: return ss2d_launch<N, CPT, 48>(p, nthreads, ctas, s);
    case 64: return ss2d_launch<N, CPT, 64>(p, nthreads, ctas, s);
  }
  set_error("sigma_ss2d_scan_fwd: dt_rank %d > 64 unsupported", p.R);
  return SIGMA_EUNSUPPORTED;
}

static int kind_dirs(int kind) { return kind == SIGMA_DIRS_CROSS4 ? 4 : (kind == SIGMA_DIRS_SEQ2 ? 2 : 1); }
static int lt_for(int N) { return N >= 16 ? Ss2dCfg<16>::LT : Ss2dCfg<4>::LT; }

// warps per CTA: a count <= maxw whose channel tile (32·cpt channels per warp) divides D, tried in the order 4, 2, 3, 1 —
// 3-warp CTAs (D = 192: 2 x 96 channels) run the four-direction scans at the same 12 resident warps per SM as 2-warp ones
// (3 x 64) with fewer, longer CTAs; ragged D falls back to enough warps to cover it with a partially filled last CTA (TMA zero-fills, y goes to the sink)
static int pick_warps(int D, int cpt, int maxw) {
  const int cpw = 32 * cpt;
  const int order[4] = {4, 2, 3, 1};
  for (int w : order)
    if (w <= maxw && D % (cpw * w) == 0) return w;
  return std::max(1, std::min(maxw, (D + cpw - 1) / cpw));
}

constexpr int kMaxSplit = 32;

// Which register budget to run (`CTAS` of ss2d_scan_kernel): the scans are MUFU / MIO-limited, so more resident warps than
// 12 buy little; d_state 16 at dt_rank 24 (stage 2, nine blocks) is the one case that runs 16.  SIGMA_SCAN_CTAS overrides.
static int ss2d_pick_ctas(int N, int rp) {
  return (N == 16 && rp == 24) ? 4 : 3;
}

// Number of L-segments for a grid of `ctas` CTAs of `nw` warps walking `ntiles` tiles each.  Model: CTAs spread evenly over the
// 132 SMs, the kernel lasts as long as its busiest SM; a warp's time per tile grows with the warps sharing its sub-partition
// (MUFU / issue are shared: per-warp cost 1 : 1.5 : 2.25 for 1 : 2 : 3 warps); a segmented walk runs two passes (summary +
// apply) and pays a fixed ring fill / parameter load per CTA (~2 tiles).  tests/test_launch_heuristics_cpu.py holds the
// model's choices to a recorded H100 sweep of every Sigma call shape x {1, 2, 4, 8} images x 10 forced counts
// (tests/golden/ss2d_split_sweep_h100.txt, scripts/bench_ss2d_splits.py).  Candidates within 3 % keep the smaller count.
static int ss2d_pick_segments(long long ctas, int nw, int ntiles, int N) {
  (void)N;                                                    // d_state 4 and 16 fit the same constants
  const double pf = 1.95;
  const int cap_warps = 12;                                   // resident warps per SM (168 registers)
  double best = 1e300;
  int best_n = 1;
  // candidate counts: the ones the recorded sweep measured (between them the model has no data to rank counts by)
  static const int kCandidates[] = {1, 2, 3, 4, 6, 8, 12, 16, 24, 32};
  for (int n : kCandidates) {
    if (n > std::min(kMaxSplit, ntiles)) break;
    const int tps = (ntiles + n - 1) / n, ne = (ntiles + tps - 1) / tps;
    if (ne != n) continue;
    const long long per_sm = (ctas * ne + kNumSMs - 1) / kNumSMs;         // CTAs on the busiest SM
    const long long warps_sm = per_sm * nw;
    const long long rounds = (warps_sm + cap_warps - 1) / cap_warps;
    const long long w_smsp = (std::min<long long>(warps_sm, cap_warps) + 3) / 4;   // warps sharing a sub-partition
    const double share = std::max(1.0, 0.75 * (double)w_smsp);
    const double cost = (double)rounds * (tps + 2) * share * (ne > 1 ? pf : 1.0);
    if (cost < best * 0.97) { best = cost; best_n = ne; }
  }
  return best_n;
}

int ss2d_pick_segments_hook(long long ctas, int nw, int ntiles, int N) { return ss2d_pick_segments(ctas, nw, ntiles, N); }

size_t ss2d_scan_workspace_bytes(int kind, int batch, int D, int N) {
  return (size_t)batch * kind_dirs(kind) * D * kMaxSplit * 2 * N * sizeof(float);
}

// The launch plan of the forward: everything ss2d_scan_fwd decides before it builds the tensor maps.  One function, so that the
// launch and its host-only query (sigma_test_ss2d_fwd_plan) cannot disagree.
struct Ss2dFwdPlan {
  int nw;                        // warps per CTA (the CTA covers 32·nw channels)
  int nsplit, tiles_per_split;   // L-segments and LT-position tiles per segment, shared by all directions
  int max_tiles, min_tiles;      // LT-position tiles of the longest / shortest direction's walk
  int nst;                       // TMA ring depth
  int rbud;                      // register budget: the `CTAS` of the ss2d_scan_kernel build that runs
  size_t smem;                   // dynamic shared memory per CTA
};

// have_ws: the caller passed a workspace of at least ss2d_scan_workspace_bytes
static int ss2d_fwd_plan(int kind, int batch, int H, int W, int D, int N, int R, int xc_dtype, int force_split, bool have_ws,
                         Ss2dFwdPlan &pl) {
  if (N != 4 && N != 8 && N != 16) {
    set_error("sigma_ss2d_scan_fwd: d_state=%d unsupported by the fused kernel (4, 8, 16)", N);
    return SIGMA_EUNSUPPORTED;
  }
  if (pad_rp(R) < 0) {
    set_error("sigma_ss2d_scan_fwd: dt_rank %d > 64 unsupported", R);
    return SIGMA_EUNSUPPORTED;
  }
  const int Cp = 2 * N + pad_rp(R);
  const int xes = xc_dtype == SIGMA_F32 ? 4 : 2;   // bytes per xc / y element
  const int ndir = kind_dirs(kind);
  const long long Lseq = kind == SIGMA_DIRS_SEQ2 ? 2LL * H * W : (long long)H * W;
  const int LT = lt_for(N);
  const int cpt = 1;   // channels per thread; CPT = 2 (shared B/C reads) lost at every Sigma shape (profiles/r01_scan_variants.txt)
  int maxw = 4;  // warps per CTA (Ss2dCfg::MAXW; the kernels' register budget assumes 128 threads)
  if (const char *e = getenv("SIGMA_SCAN_WARPS")) maxw = std::max(1, std::min(4, atoi(e)));
  const int NW = pick_warps(D, cpt, maxw), DT = 32 * cpt * NW;
  int max_tiles = 0, min_tiles = 0;
  for (int k = 0; k < ndir; ++k) {
    const bool colmajor = kind == SIGMA_DIRS_CROSS4 && (k & 1);
    const long long I = colmajor ? H : Lseq, O = colmajor ? W : 1;
    const int nt = (int)(O * ((I + LT - 1) / LT));
    max_tiles = std::max(max_tiles, nt);
    min_tiles = k == 0 ? nt : std::min(min_tiles, nt);
  }
  // L-segments (MODE_SUMMARY -> combine -> MODE_APPLY): a second pass over the data, so only when the unsplit grid leaves SM
  // sub-partitions without a warp.  ss2d_pick_segments models the busiest SM (the old rule, "fill 592 warp slots", ignored
  // wave quantisation: 312 CTAs of 2 warps put 6 warps on some SMs where 288 put 4 on every SM).  SIGMA_SCAN_SPLIT_RULE=old
  // restores the round-1 rule for comparison.
  const long long ctas = (long long)((D + DT - 1) / DT) * ndir * batch;
  const long long warps = ctas * NW;
  const long long full = kNumSMs * 4;
  int nsplit = 1;
  const char *rule = getenv("SIGMA_SCAN_SPLIT_RULE");
  if (rule && rule[0] == 'o') {
    if (warps < full) {
      const long long want = N >= 16 ? full : 2 * full;
      nsplit = (int)std::min<long long>((want + warps - 1) / warps, kMaxSplit);
    }
  } else if (warps < 3 * full) {
    nsplit = ss2d_pick_segments(ctas, NW, max_tiles, N);
  }
  if (force_split > 0) nsplit = std::min(force_split, kMaxSplit);
  if (!have_ws) {
    if (force_split > 1) { set_error("sigma_ss2d_scan_fwd: workspace too small for %d segments", force_split); return SIGMA_EWORKSPACE; }
    nsplit = 1;
  }
  nsplit = std::max(1, std::min(nsplit, max_tiles));
  // all directions share tiles_per_split; directions with fewer tiles simply get empty trailing segments
  pl.tiles_per_split = (max_tiles + nsplit - 1) / nsplit;
  pl.nsplit = nsplit;
  pl.max_tiles = max_tiles;
  pl.min_tiles = min_tiles;
  pl.nw = NW;

  // register budget (ss2d_scan.cuh): which `__launch_bounds__(128, CTAS)` build runs.  SIGMA_SCAN_CTAS overrides.
  int rbud = ss2d_pick_ctas(N, pad_rp(R));
  if (const char *e = getenv("SIGMA_SCAN_CTAS")) rbud = std::max(3, std::min(5, atoi(e)));
  if (N != 16 || xc_dtype != SIGMA_F32) rbud = 3;   // bf16 / fp16: only the 3-CTA budget is built (ss2d_scan_inst.inc)
  rbud = std::min(rbud, 4);
  pl.rbud = rbud;
  {
    // TMA ring depth: as many stages as fit without lowering the register-limited occupancy (227 KB per SM, 1 KB
    // reserved per CTA).
    // Deep rings matter: a tile is requested when the LAST warp releases its slot and needed by the FIRST warp
    // nst-1 tiles later; with 3-4 stages the warps spun on the full barrier ~80 times per tile (ncu, round 1).
    const size_t stage = (size_t)LT * DT * xes + (size_t)LT * Cp * (kind == SIGMA_DIRS_CROSS ? 2 : 1) * sizeof(float);
    // resident CTAs per SM by registers (e.g. 168 per thread under __launch_bounds__(128, 3): 3 / 4 / 6 / 12 for 4 / 3 / 2 / 1 warps)
    const int ctas_sm = std::max(rbud, std::min(16, 65536 / (32 * NW * ss2d_reg_cap(rbud))));
    const size_t budget = (227 * 1024) / ctas_sm - 1024 - 128;
    pl.nst = (int)std::max<size_t>(2, std::min<size_t>(Ss2dCfg<16>::MAX_NST, budget / stage));
    if (const char *e = getenv("SIGMA_SCAN_NST")) pl.nst = std::max(2, std::min(Ss2dCfg<16>::MAX_NST, atoi(e)));
  }
  pl.smem = ss2d_smem_bytes(LT, DT, pl.nst, Cp, kind == SIGMA_DIRS_CROSS, xes);
  return SIGMA_OK;
}

int ss2d_fwd_plan_hook(int kind, int batch, int H, int W, int D, int N, int R, int xc_dtype, int force_split, size_t ws_bytes,
                       long long *out8) {
  Ss2dFwdPlan pl;
  const bool have_ws = ws_bytes > 0 && ws_bytes >= ss2d_scan_workspace_bytes(kind, batch, D, N);
  const int rc = ss2d_fwd_plan(kind, batch, H, W, D, N, R, xc_dtype, force_split, have_ws, pl);
  if (rc) return rc;
  const long long v[8] = {pl.nsplit, pl.tiles_per_split, pl.max_tiles, pl.min_tiles, pl.nw, pl.nst, pl.rbud, (long long)pl.smem};
  for (int i = 0; i < 8; ++i) out8[i] = v[i];
  return SIGMA_OK;
}

// xc_dtype SIGMA_BF16 / SIGMA_F16: xc and y are bf16 / fp16 (passed through the float pointers); x_dbl, the parameters and the
// recurrence stay fp32
int ss2d_scan_fwd(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                  const float *Ds, float *y, int batch, int H, int W, int D, int N, int R, int Cp, void *ws,
                  size_t ws_bytes, int force_split, cudaStream_t stream, float *dsave, float *hsave, int xc_dtype) {
  Ss2dFwdPlan pl;
  int rc = ss2d_fwd_plan(kind, batch, H, W, D, N, R, xc_dtype, force_split,
                         ws != nullptr && ws_bytes >= ss2d_scan_workspace_bytes(kind, batch, D, N), pl);
  if (rc) return rc;
  Ss2dParams p;
  memset(&p, 0, sizeof(p));
  p.xc_dtype = xc_dtype;
  const int xes = xc_dtype == SIGMA_F32 ? 4 : 2;   // bytes per xc / y element
  const CUtensorMapDataType xdt = xc_dtype == SIGMA_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                  : xc_dtype == SIGMA_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  p.dtw = dtw; p.dtb = dtb; p.A = A; p.Ds = Ds; p.y = y; p.carry = (float *)ws;
  p.D = D; p.N = N; p.R = R; p.Cp = Cp; p.kind = kind; p.batch = batch;
  p.dsave = dsave; p.hsave = hsave; p.save_tiles = hsave ? ss2d_save_tiles(kind, H, W) : 0;
  const int ndir = kind_dirs(kind);
  p.ndir = ndir;
  if (const char *e = getenv("SIGMA_SCAN_ABLATE")) p.ablate = atoi(e);
  const int K = kind == SIGMA_DIRS_CROSS ? 1 : ndir;        // x_dbl rows per position
  const long long Lseq = kind == SIGMA_DIRS_SEQ2 ? 2LL * H * W : (long long)H * W;
  p.Lseq = Lseq;
  const int LT = lt_for(N);
  const int NW = pl.nw, DT = 32 * NW;
  for (int k = 0; k < ndir; ++k) {
    const bool colmajor = kind == SIGMA_DIRS_CROSS4 && (k & 1);
    p.rev[k] = (kind == SIGMA_DIRS_CROSS4) ? (k >= 2) : (kind == SIGMA_DIRS_SEQ2 ? (k == 1) : 0);
    uint64_t dims[4], str[3];
    uint32_t box[4] = {(uint32_t)DT, (uint32_t)LT, 1, 1};
    // channels-last activations (batch, Lseq, D)
    if (!colmajor) {
      p.I[k] = (int)Lseq; p.O[k] = 1;
      p.istride[k] = D; p.ostride[k] = 0;
      dims[0] = D; dims[1] = Lseq; dims[2] = 1; dims[3] = batch;
      str[0] = (uint64_t)D * xes; str[1] = (uint64_t)Lseq * D * xes; str[2] = (uint64_t)Lseq * D * xes;
    } else {  // walk h (inner) at fixed w (outer): l1 = w·H + h  <->  position h·W + w   (vmamba.py:87)
      p.I[k] = H; p.O[k] = W;
      p.istride[k] = (long long)W * D; p.ostride[k] = D;
      dims[0] = D; dims[1] = H; dims[2] = W; dims[3] = batch;
      str[0] = (uint64_t)W * D * xes; str[1] = (uint64_t)D * xes; str[2] = (uint64_t)Lseq * D * xes;
    }
    if ((rc = make_tmap(&p.m_xc[k], xdt, 4, xc, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B)))
      return rc;
    // x_dbl (batch, Lseq, K, Cp): direction k's row starts at column k·Cp
    uint32_t boxd[4] = {(uint32_t)Cp, (uint32_t)LT, 1, 1};
    dims[0] = Cp;
    const uint64_t pos = (uint64_t)K * Cp * 4;
    if (!colmajor) { str[0] = pos; str[1] = Lseq * pos; str[2] = Lseq * pos; }
    else { str[0] = W * pos; str[1] = pos; str[2] = Lseq * pos; }
    if ((rc = make_tmap(&p.m_dbl[k], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, xdbl + (long long)(kind == SIGMA_DIRS_CROSS ? 0 : k) * Cp, dims,
                        str, boxd, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))) return rc;
  }
  p.tiles_per_split = pl.tiles_per_split;
  p.nsplit = pl.nsplit;
  p.nst = pl.nst;
  const int nthreads = 32 * NW;
  switch (N) {
    case 4: return dispatch_rp<4, 1>(p, nthreads, pl.rbud, stream);
    case 8: return dispatch_rp<8, 1>(p, nthreads, pl.rbud, stream);
    case 16: return dispatch_rp<16, 1>(p, nthreads, pl.rbud, stream);
  }
  set_error("sigma_ss2d_scan_fwd: d_state=%d unsupported by the fused kernel (4, 8, 16)", N);
  return SIGMA_EUNSUPPORTED;
}

}  // namespace sigma
