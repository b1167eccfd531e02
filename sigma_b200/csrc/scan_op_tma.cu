// a1 — op-level selective scan forward on the fused kernel's machinery, for the reference layout
// (reference: csrc/selective_scan/selective_scan.cpp:165-249, selective_scan_fwd_kernel.cuh:64-206).
//
// One thread owns one channel with all N states in registers (no shuffles); a warp = 32 consecutive channels of one
// (batch, group); a CTA = up to 4 warps.  u / delta tiles ({64 B of L} x DT channels) and the group's B / C tiles arrive
// through a TMA ring (one "full" mbarrier per slot; the LAST warp to finish a tile requests the tile that reuses its
// slot — no producer warp, no CTA barrier in the loop).  Each warp transposes B / C into its private fp32
// [position][B | C] tile (scan_op_tma.cuh), runs the state-pair recurrence of the fused kernel with the delta'
// (bias + softplus) of the NEXT group of positions issued next to the current group's exponentials, writes y IN PLACE
// over its u rows (same element type) and stores its 32 rows with ONE TMA store per tile.  fp16 / bf16 are loaded and
// stored natively (no cast passes).  L-segments (MODE_SUMMARY -> combine -> MODE_APPLY) as in the fused kernel when
// the grid cannot fill the machine.  Shapes TMA cannot express (rows not 16-byte aligned, channel groups not a multiple
// of 32, d_state > 16) take the generic kernel in scan_op.cu.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <unordered_set>

#include "scan_op_tma.cuh"

namespace sigma {

// Opt a kernel into the full 227 KB of dynamic shared memory, once per kernel and process (cudaFuncSetAttribute on every
// call was a measurable part of the small-batch launch floor).
cudaError_t prep_kernel_once(const void *fn) {
  static std::mutex mu;
  static std::unordered_set<const void *> seen;
  std::lock_guard<std::mutex> lk(mu);
  if (seen.count(fn)) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e == cudaSuccess) seen.insert(fn);
  return e;
}

struct alignas(64) ScanTmaParams {
  CUtensorMap m_u, m_dl, m_B, m_C, m_out;
  const float *A, *D, *bias;
  float *x, *hs, *carry;
  long long A_d, A_n;
  int batch, dim, L, N, G, dpg, ctiles_per_group, DT, softplus;
  int nsplit, tiles_per_split, ntiles, nchunks, nst, nhs;
};

template <int NP> struct OpCfg {
  static constexpr int G = NP >= 16 ? 4 : 8;      // positions per software-pipelined group (as the fused kernel)
  static constexpr int CTAS = NP >= 16 ? 3 : 4;   // resident 128-thread CTAs per SM the register budget allows
};

template <typename T, int NP>
__host__ __device__ constexpr int op_bct_floats() { return OpT<T>::LT * (2 * NP + 4); }

template <typename T, int NP>
__host__ __device__ inline size_t op_tma_smem_bytes(int DT, int nst) {
  const size_t stage = (size_t)2 * DT * OPT_ROW_BYTES + (size_t)2 * NP * OPT_ROW_BYTES;
  return 1024 /*alignment slack*/ + nst * stage + (size_t)(DT / 32) * op_bct_floats<T, NP>() * sizeof(float) + 256;
}

// YOUT = false: no C / y / store — MODE_SUMMARY (segment summaries) or the state-only sweep of the backward (`hs`).
template <typename T, int NP, int MODE, bool YOUT>
__global__ void __launch_bounds__(128, OpCfg<NP>::CTAS) scan_op_tma_kernel(const __grid_constant__ ScanTmaParams p) {
  constexpr int LT = OpT<T>::LT, G = OpCfg<NP>::G, NG = LT / G, PITCH = 2 * NP + 4;
  constexpr bool WITH_Y = YOUT;
  static_assert(!(MODE == MODE_SUMMARY && YOUT), "summary pass has no output");
  constexpr int NCH = NP >= 8 ? 2 : 1;

  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char *smem = reinterpret_cast<unsigned char *>(((uintptr_t)smem_dyn + 1023) & ~(uintptr_t)1023);
  const int DT = p.DT, NST = p.nst;
  const int u_b = DT * OPT_ROW_BYTES, bc_b = NP * OPT_ROW_BYTES, stage_b = 2 * u_b + 2 * bc_b;
  float *bct_all = reinterpret_cast<float *>(smem + (size_t)NST * stage_b);
  uint64_t *full = reinterpret_cast<uint64_t *>(bct_all + (DT / 32) * op_bct_floats<T, NP>());
  uint32_t *done = reinterpret_cast<uint32_t *>(full + NST);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = DT >> 5;
  const int g = blockIdx.x / p.ctiles_per_group, ct = blockIdx.x - g * p.ctiles_per_group;
  const int d0 = g * p.dpg + ct * DT, d = d0 + tid;
  const int b = blockIdx.z, split = blockIdx.y;
  const int t0 = split * p.tiles_per_split, t1 = min(p.ntiles, t0 + p.tiles_per_split);

  if (tid == 0) {
    for (int s = 0; s < NST; ++s) { mbar_init(&full[s], 1); done[s] = 0; }
    fence_mbar_init();
  }
  __syncthreads();

  const uint32_t tx_bytes = (uint32_t)stage_b;
  auto request_tile = [&](int tau, int st) {
    unsigned char *dst = smem + (size_t)st * stage_b;
    const int l0 = tau * LT;
    mbar_arrive_expect_tx(&full[st], tx_bytes);
    tma_load_3d(dst, &p.m_u, &full[st], l0, d0, b);
    tma_load_3d(dst + u_b, &p.m_dl, &full[st], l0, d0, b);
    tma_load_4d(dst + 2 * u_b, &p.m_B, &full[st], l0, 0, g, b);
    tma_load_4d(dst + 2 * u_b + bc_b, &p.m_C, &full[st], l0, 0, g, b);
  };
  if (tid == 0) {
    tma_prefetch_desc(&p.m_u); tma_prefetch_desc(&p.m_dl); tma_prefetch_desc(&p.m_B); tma_prefetch_desc(&p.m_C);
    if (WITH_Y) tma_prefetch_desc(&p.m_out);
    for (int tau = t0; tau < min(t1, t0 + NST); ++tau) request_tile(tau, tau - t0);
  }

  // ---- per-thread constants: one channel, all states ----
  float h[NP], a2[NP];
#pragma unroll
  for (int s = 0; s < NP; ++s) {
    a2[s] = s < p.N ? p.A[(long long)d * p.A_d + (long long)s * p.A_n] * kLog2e : 0.f;
    h[s] = 0.f;
  }
  const float bias = p.bias ? p.bias[d] : 0.f;
  const float Dv = p.D ? p.D[d] : 0.f;
  const bool sp = p.softplus != 0;
  float sumdl = 0.f;      // Σ delta' over this CTA's walk (running prefix of the chunk states; segment product in MODE_SUMMARY)
  // (prod a, h) of this CTA's L-segment: written by MODE_SUMMARY, chained by the combine kernel, read by MODE_APPLY
  auto carry_row = [&]() { return p.carry + (((long long)b * p.dim + d) * p.nsplit + split) * 2 * NP; };
  if (MODE == MODE_APPLY) {
    const float *cr = carry_row();
#pragma unroll
    for (int s = 0; s < NP; ++s) h[s] = cr[NP + s];
  }
  float *bct = bct_all + warp * op_bct_floats<T, NP>();

  int st = 0, ph = 0, pst = 0;
  for (int tau = t0; tau < t1; ++tau) {
    mbar_spin(&full[st], (uint32_t)ph);
    unsigned char *sU = smem + (size_t)st * stage_b;
    const unsigned char *sDl = sU + u_b;
    __syncwarp();   // every lane is done reading the previous tile's B / C rows
    transpose_bc<T, NP>(sU + 2 * u_b, sU + 2 * u_b + bc_b, bct, lane);
    __syncwarp();
    const int npos = min(LT, p.L - tau * LT);
    const int ng = (npos + G - 1) / G;

    float dl[G], u[G];
    {
      float raw[G];
      load_group<T, G>(sDl, tid, 0, raw);
      load_group<T, G>(sU, tid, 0, u);
#pragma unroll
      for (int i = 0; i < G; i += 2) {   // softplus of two positions per call (G is even)
        const float r0 = raw[i] + bias, r1 = raw[i + 1] + bias;
        const f2 s2 = sp ? softplus20x2(r0, r1) : f2{r0, r1};
        dl[i] = s2.x; dl[i + 1] = s2.y;
      }
    }
#pragma unroll 1
    for (int gi = 0; gi < ng; ++gi) {
      if (MODE != MODE_SUMMARY && p.hs != nullptr && (gi * G) % OPT_HS_POS == 0) {   // state checkpoints for the backward
        float4 *hrow = reinterpret_cast<float4 *>(p.hs + (((long long)b * p.dim + d) * p.nhs + (tau * LT + gi * G) / OPT_HS_POS) * NP);
#pragma unroll
        for (int q = 0; q < NP / 4; ++q) hrow[q] = make_float4(h[4 * q], h[4 * q + 1], h[4 * q + 2], h[4 * q + 3]);
      }
      // next group's delta' / u first: its loads and softplus overlap this group's exponentials
      float dln[G], un[G];
      {
        const int gn = gi + 1 < NG ? gi + 1 : gi;
        float raw[G];
        load_group<T, G>(sDl, tid, gn, raw);
        load_group<T, G>(sU, tid, gn, un);
#pragma unroll
        for (int i = 0; i < G; i += 2) {
          const float r0 = raw[i] + bias, r1 = raw[i + 1] + bias;
          const f2 s2 = sp ? softplus20x2(r0, r1) : f2{r0, r1};
          dln[i] = s2.x; dln[i + 1] = s2.y;
        }
      }
      const int cnt = npos - gi * G;      // valid positions of this group (>= 1)
      float yv[G];
      // one position of the recurrence: B / C of the position are 2·NP/4 broadcast LDS.128; per state pair FMUL2 (exp
      // arguments), 2 x MUFU.EX2, mul2 (delta·u·B), fma2 (h), fma2 (C·h)
      auto position = [&](int i) {
        const float *row = bct + (gi * G + i) * PITCH;
        const float dd = dl[i], du = dl[i] * u[i];
        f2 yacc[NCH];
#pragma unroll
        for (int s4 = 0; s4 < NP / 4; ++s4) {
          const float4 bv = *reinterpret_cast<const float4 *>(row + 4 * s4);
          float4 cv = make_float4(0.f, 0.f, 0.f, 0.f);
          if (WITH_Y) cv = *reinterpret_cast<const float4 *>(row + NP + 4 * s4);
#pragma unroll
          for (int hp = 0; hp < 2; ++hp) {
            const int s = 4 * s4 + 2 * hp;
            const f2 arg = mul2(f2{dd, dd}, f2{a2[s], a2[s + 1]});
            const f2 a = f2{ex2(arg.x), ex2(arg.y)};
            const f2 bb = mul2(f2{du, du}, hp == 0 ? f2{bv.x, bv.y} : f2{bv.z, bv.w});
            const f2 hn = fma2(a, f2{h[s], h[s + 1]}, bb);
            h[s] = hn.x; h[s + 1] = hn.y;
            if (WITH_Y) {
              const f2 cc = hp == 0 ? f2{cv.x, cv.y} : f2{cv.z, cv.w};
              const int ch = NCH == 2 ? hp : 0;
              const bool first = NCH == 2 ? s4 == 0 : (s4 == 0 && hp == 0);
              yacc[ch] = first ? mul2(hn, cc) : fma2(hn, cc, yacc[ch]);
            }
          }
        }
        if (WITH_Y) {
          float y = yacc[0].x + yacc[0].y;
          if (NCH == 2) y += yacc[1].x + yacc[1].y;
          yv[i] = fmaf(Dv, u[i], y);
        }
        sumdl += dd;
      };
      if (cnt >= G) {   // full group: one basic block, the prologue above interleaves with it
#pragma unroll
        for (int i = 0; i < G; ++i) position(i);
      } else {          // ragged end of the sequence: positions past L must not advance the state (TMA zero-filled them)
#pragma unroll
        for (int i = 0; i < G; ++i) {
          yv[i] = 0.f;
          if (i < cnt) position(i);
        }
      }
      if (WITH_Y) store_group<T, G>(sU, tid, gi, yv);   // y over u, in place (same rows, same swizzle)
#pragma unroll
      for (int i = 0; i < G; ++i) { dl[i] = dln[i]; u[i] = un[i]; }
    }

    if (WITH_Y) {
      // chunk-end states (prod a since the sequence start, h) every 2048 positions (selective_scan_fwd_kernel.cuh:181-184)
      if (p.x != nullptr) {
        const int lend = tau * LT + npos;
        if ((lend & 2047) == 0 || lend == p.L) {
          const int c = (lend - 1) >> 11;
          float *xr = p.x + (((long long)b * p.dim + d) * p.nchunks + c) * 2 * p.N;
#pragma unroll
          for (int s = 0; s < NP; ++s) {
            if (s < p.N) {
              float P = ex2(a2[s] * sumdl);
              if (MODE == MODE_APPLY) P *= carry_row()[s];   // product over the preceding segments
              xr[2 * s] = P;
              xr[2 * s + 1] = h[s];
            }
          }
        }
      }
      // this warp's 32 rows of y -> global: generic-proxy writes made visible to the async proxy, one TMA store.  The
      // slot is released one tile LATER (when at most one store group is still reading shared memory): nobody waits for
      // a TMA store, the ring is one stage deeper instead.
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        tma_store_3d(&p.m_out, sU + warp * 32 * OPT_ROW_BYTES, tau * LT, d0 + warp * 32, b);
        tma_store_commit();
        if (tau > t0) {
          tma_store_wait_read<1>();
          if (tau - 1 + NST < t1) {
            const uint32_t old = smem_inc_acq_rel(&done[pst]);
            if ((old + 1) % (uint32_t)nwarps == 0) request_tile(tau - 1 + NST, pst);
          }
        }
      }
      __syncwarp();
    } else {
      __syncwarp();
      if (lane == 0 && tau + NST < t1) {
        const uint32_t old = smem_inc_acq_rel(&done[st]);
        if ((old + 1) % (uint32_t)nwarps == 0) request_tile(tau + NST, st);
      }
    }
    pst = st;
    if (++st == NST) { st = 0; ph ^= 1; }
  }
  if (WITH_Y && lane == 0) tma_store_wait_all<0>();

  if (MODE == MODE_SUMMARY) {
    float *cr = carry_row();
#pragma unroll
    for (int s = 0; s < NP; ++s) {
      cr[s] = ex2(a2[s] * sumdl);
      cr[NP + s] = h[s];
    }
  }
}

// ---- host side ----
constexpr int kOpMaxSplit = 64;

size_t scan_op_tma_workspace_bytes(int batch, int dim, int dstate) {
  const int NP = dstate <= 4 ? 4 : (dstate <= 8 ? 8 : 16);
  return (size_t)batch * dim * kOpMaxSplit * 2 * NP * sizeof(float);
}

// Number of L-segments minimising  waves x (tiles per segment + fixed) x passes  over 1..max_split: `slots` = CTAs resident on the
// whole GPU, `pass_factor` = cost of summary + apply relative to one unsplit sweep.
int pick_segments(long long ctas_base, int ntiles, long long slots, double pass_factor, int max_split) {
  double best = 1e300;
  int best_n = 1;
  for (int n = 1; n <= std::min(max_split, ntiles); ++n) {
    const int tps = (ntiles + n - 1) / n, ne = (ntiles + tps - 1) / tps;
    if (ne != n) continue;
    const long long waves = (ctas_base * ne + slots - 1) / slots;
    const double cost = (double)waves * (tps + 3) * (ne > 1 ? pass_factor : 1.0);
    if (cost < best * 0.97) { best = cost; best_n = ne; }   // a larger count must win by > 3 %
  }
  return best_n;
}

template <typename T>
bool scan_op_tma_eligible(const void *u, const void *delta, const void *B, const void *C, const void *out, int dim, int L,
                          int N, int G, const sigma_scan_strides &s) {
  if (!(N == 4 || N == 8 || N == 16)) return false;
  if ((dim / G) % 32 != 0) return false;
  const long long sz = sizeof(T);
  auto al = [&](const void *ptr) { return ((uintptr_t)ptr & 15) == 0; };
  auto ok = [&](long long stride_elems) { return stride_elems > 0 && (stride_elems * sz) % 16 == 0; };
  if (!(al(u) && al(delta) && al(B) && al(C) && al(out))) return false;
  if (!(ok(s.u_dim) && ok(s.delta_dim) && ok(s.out_dim) && ok(s.B_dstate) && ok(s.C_dstate) && ok(s.B_group) && ok(s.C_group)))
    return false;
  if (!(ok(s.u_batch) && ok(s.delta_batch) && ok(s.out_batch) && ok(s.B_batch) && ok(s.C_batch))) return false;
  if ((long long)L * sz < 16) return false;
  return true;
}

template <typename T, int NP>
static int launch_tma(ScanTmaParams &p, bool yout, cudaStream_t stream) {
  const size_t smem = op_tma_smem_bytes<T, NP>(p.DT, p.nst);
  dim3 grid(p.G * p.ctiles_per_group, p.nsplit, p.batch), block(p.DT);
  auto prep = [&](const void *fn) -> cudaError_t { return prep_kernel_once(fn); };
  auto run = [&](auto kern) -> int {
    SIGMA_CHECK_CUDA(prep((const void *)kern));
    kern<<<grid, block, smem, stream>>>(p);
    SIGMA_CHECK_LAUNCH();
    return SIGMA_OK;
  };
  int rc;
  if (p.nsplit == 1) return yout ? run(scan_op_tma_kernel<T, NP, MODE_SERIAL, true>) : run(scan_op_tma_kernel<T, NP, MODE_SERIAL, false>);
  if ((rc = run(scan_op_tma_kernel<T, NP, MODE_SUMMARY, false>))) return rc;
  const long long nrows = (long long)p.batch * p.dim, tot = nrows * NP;
  scan_combine_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(p.carry, nrows, p.nsplit, NP);
  SIGMA_CHECK_LAUNCH();
  return yout ? run(scan_op_tma_kernel<T, NP, MODE_APPLY, true>) : run(scan_op_tma_kernel<T, NP, MODE_APPLY, false>);
}

// Launch plan of scan_op_fwd_tma (host only; eligibility guarantees N in {4, 8, 16} and dim / G a multiple of 32).  16-bit
// elements have 32-position tiles, fp32 16-position ones.
ScanOpPlan scan_op_fwd_tma_plan(int elem_bytes, int batch, int dim, int L, int N, int G, bool have_ws, int force_split) {
  const int LT = elem_bytes == 4 ? OpT<float>::LT : OpT<__half>::LT, NP = N, dpg = dim / G;
  ScanOpPlan pl;
  // channels per CTA: the largest of 128 / 96 / 64 / 32 that divides the group
  pl.DT = 32;
  for (int w = 4; w >= 1; --w)
    if (dpg % (32 * w) == 0) { pl.DT = 32 * w; break; }
  pl.ntiles = (L + LT - 1) / LT;

  // L-segments (MODE_SUMMARY -> combine -> MODE_APPLY).  Model: a
  // tile costs about the same 3-5 us whether 1 or 3 warps share an SM sub-partition (latency-bound alone, MUFU-bound together),
  // so time ~ waves x tiles-per-segment x passes: pick the segment count that minimises that, i.e. fills whole waves of the
  // resident CTA slots.  Segments need not end on the 2048-position chunk boundaries of `x`: a segment that crosses one writes
  // that chunk's state itself (true h, prefix product = carry-in x local).
  const long long ctas_base = (long long)batch * G * (dpg / pl.DT);
  int nsplit = pick_segments(ctas_base, pl.ntiles, kNumSMs * (N >= 16 ? 3 : 4) * 4 / (pl.DT / 32), 2.2, kOpMaxSplit);
  if (force_split > 0) nsplit = std::min(force_split, kOpMaxSplit);
  if (!have_ws) nsplit = 1;
  const int tps = std::max(1, (pl.ntiles + nsplit - 1) / nsplit);
  pl.tiles_per_split = tps;
  pl.nsplit = std::max(1, (pl.ntiles + tps - 1) / tps);

  // ring depth: what fits next to the other resident CTAs
  {
    const int nw = pl.DT / 32;
    const int regs_ctas = std::min(NP >= 16 ? 12 / nw : 16 / nw, 16);          // 12 / 16 resident warps per SM by registers
    const size_t budget = (size_t)(227 * 1024) / std::max(1, regs_ctas) - 1024;
    const size_t stage = (size_t)2 * pl.DT * OPT_ROW_BYTES + (size_t)2 * NP * OPT_ROW_BYTES;
    const size_t fixed = 1024 + 256 + (size_t)nw * LT * (2 * NP + 4) * sizeof(float);
    int nst = budget > fixed ? (int)((budget - fixed) / stage) : 2;
    pl.nst = std::max(3, std::min(8, nst));   // >= 3: a slot is released one tile after its last use
    if (const char *e = getenv("SIGMA_OP_NST")) pl.nst = std::max(3, std::min(8, atoi(e)));
  }
  return pl;
}

// `hs` (nullable): state at the start of every OPT_HS_POS positions, (batch, dim, ceil(L / OPT_HS_POS), NP) fp32.  out == nullptr: state-only
// sweep (no y), the first half of the backward.
template <typename T>
int scan_op_fwd_tma(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                    const float *bias, void *out, float *x, float *hs, int batch, int dim, int L, int N, int G, int softplus,
                    const sigma_scan_strides &s, void *ws, size_t ws_bytes, int force_split, cudaStream_t stream) {
  constexpr int LT = OpT<T>::LT;
  const int NP = N;   // eligibility guarantees N in {4, 8, 16}
  ScanTmaParams p;
  memset(&p, 0, sizeof(p));
  p.A = A; p.D = D; p.bias = bias; p.x = x; p.hs = hs; p.carry = (float *)ws;
  p.A_d = s.A_dim; p.A_n = s.A_dstate;
  p.batch = batch; p.dim = dim; p.L = L; p.N = N; p.G = G; p.dpg = dim / G; p.softplus = softplus;
  const bool have_ws = ws != nullptr && ws_bytes >= scan_op_tma_workspace_bytes(batch, dim, N);
  const ScanOpPlan pl = scan_op_fwd_tma_plan((int)sizeof(T), batch, dim, L, N, G, have_ws, force_split);
  p.DT = pl.DT;
  p.ctiles_per_group = p.dpg / p.DT;
  p.ntiles = pl.ntiles;
  p.nchunks = (L + 2047) / 2048;
  p.nhs = (L + OPT_HS_POS - 1) / OPT_HS_POS;
  p.tiles_per_split = pl.tiles_per_split;
  p.nsplit = pl.nsplit;
  p.nst = pl.nst;

  const uint64_t sz = sizeof(T);
  int rc;
  {
    uint64_t dims[3] = {(uint64_t)L, (uint64_t)dim, (uint64_t)batch};
    uint32_t box[3] = {(uint32_t)LT, (uint32_t)p.DT, 1};
    uint64_t st_u[2] = {(uint64_t)s.u_dim * sz, (uint64_t)s.u_batch * sz};
    uint64_t st_d[2] = {(uint64_t)s.delta_dim * sz, (uint64_t)s.delta_batch * sz};
    uint64_t st_o[2] = {(uint64_t)s.out_dim * sz, (uint64_t)s.out_batch * sz};
    if ((rc = make_tmap(&p.m_u, OpT<T>::kType, 3, u, dims, st_u, box, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if ((rc = make_tmap(&p.m_dl, OpT<T>::kType, 3, delta, dims, st_d, box, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    uint32_t boxo[3] = {(uint32_t)LT, 32, 1};
    if (out != nullptr &&
        (rc = make_tmap(&p.m_out, OpT<T>::kType, 3, out, dims, st_o, boxo, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE))) return rc;
    uint64_t dimb[4] = {(uint64_t)L, (uint64_t)N, (uint64_t)G, (uint64_t)batch};
    uint32_t boxb[4] = {(uint32_t)LT, (uint32_t)NP, 1, 1};
    uint64_t st_B[3] = {(uint64_t)s.B_dstate * sz, (uint64_t)s.B_group * sz, (uint64_t)s.B_batch * sz};
    uint64_t st_C[3] = {(uint64_t)s.C_dstate * sz, (uint64_t)s.C_group * sz, (uint64_t)s.C_batch * sz};
    if ((rc = make_tmap(&p.m_B, OpT<T>::kType, 4, B, dimb, st_B, boxb, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if ((rc = make_tmap(&p.m_C, OpT<T>::kType, 4, C, dimb, st_C, boxb, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
  }
  switch (NP) {
    case 4: return launch_tma<T, 4>(p, out != nullptr, stream);
    case 8: return launch_tma<T, 8>(p, out != nullptr, stream);
    default: return launch_tma<T, 16>(p, out != nullptr, stream);
  }
}

#define SIGMA_INST(T)                                                                                                           \
  template bool scan_op_tma_eligible<T>(const void *, const void *, const void *, const void *, const void *, int, int, int,   \
                                        int, const sigma_scan_strides &);                                                      \
  template int scan_op_fwd_tma<T>(const void *, const void *, const float *, const void *, const void *, const float *,         \
                                  const float *, void *, float *, float *, int, int, int, int, int, int,                       \
                                  const sigma_scan_strides &, void *, size_t, int, cudaStream_t);
SIGMA_INST(float)
SIGMA_INST(__half)
SIGMA_INST(__nv_bfloat16)
#undef SIGMA_INST

}  // namespace sigma
