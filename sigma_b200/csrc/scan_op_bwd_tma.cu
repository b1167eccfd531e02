// a3 — op-level selective scan backward, TMA-staged, for the reference layout
// (reference: csrc/selective_scan/selective_scan.cpp:251-362, selective_scan_bwd_kernel.cuh:68-274).
//
// Sweeps (all on the tile geometry of scan_op_tma.cuh: 64 bytes of L per row):
//   1. state sweep  — the forward kernel without C / y (scan_op_tma.cu, YOUT = false) leaves the state at the start of
//      every tile in scratch `hs` (the reference recomputes from its 2048-chunk states, bwd_kernel.cuh:114-116);
//   2. (only when the grid cannot fill the machine) reverse summaries per L-segment: (prod a, sum of the reverse
//      recurrence from 0) -> chained right-to-left by scan_combine_rev_kernel -> every segment knows the dh entering it;
//   3. this kernel walks its tiles BACKWARDS: per tile it recomputes h at every position from the tile's start state
//      (kept in shared memory, float4 per thread and state quad), then runs the reverse recurrence
//          dh_l = a_{l+1}·dh_{l+1} + dout_l·C_l
//      producing du, ddelta (softplus' applied; written IN PLACE over the u / delta tiles and stored by TMA), per-thread
//      dA / dD / ddelta_bias, and dB / dC: each (n, l) term is summed over the warp's channels with a transposing
//      shuffle reduction (NS/2 + NS/4 + ... shuffles instead of 5 per value) and leaves the warp as ONE vector
//      red.global.add.v4.f32 per state and 4 positions — the reference issues one scalar atomic per CHANNEL per (n, l)
//      (bwd_kernel.cuh:214-227).
// Mapping: d_state 16 -> 2 lanes per channel (8 states each, lanes l and l+16 of a warp); d_state <= 8 -> 1 lane per
// channel.  A CTA covers 64 (or 32) channels of one (batch, group).
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "scan_op_tma.cuh"

namespace sigma {

struct alignas(64) ScanBwdTmaParams {
  CUtensorMap m_u, m_dl, m_do, m_B, m_C, m_du, m_dd;
  const float *A, *D, *bias, *hs;
  float *dA, *dB, *dC, *dD, *dbias, *carry;
  int batch, dim, L, N, G, dpg, ctiles_per_group, DT, softplus;
  int nsplit, tiles_per_split, ntiles, nst, nhs;
  // deterministic build (scan_op_bwd_tma_det_kernel): dB / dC partials per warp channel tile of a group (dpg / CPW, batch, G,
  // N, L); dA (batch·nsplit, dim, N), dD and ddelta_bias (batch·nsplit, dim) per (batch, L-segment)
  float *part_B, *part_C, *part_dA, *part_dD, *part_db;
};

template <int NP> struct BwdCfg {
  static constexpr int LPC = NP >= 16 ? 2 : 1;   // lanes per channel
  static constexpr int NS = NP / LPC;            // states per lane
  static constexpr int CPW = 32 / LPC;           // channels per warp
};

template <typename T, int NP>
__host__ __device__ inline size_t bwd_tma_smem_bytes(int DT, int nst) {
  constexpr int LT = OpT<T>::LT, LPC = BwdCfg<NP>::LPC, NS = BwdCfg<NP>::NS;
  const int NT = DT * LPC;
  const size_t stage = (size_t)3 * DT * OPT_ROW_BYTES + (size_t)2 * NP * OPT_ROW_BYTES;
  const size_t bct = (size_t)(NT / 32) * LT * (2 * NP + 4) * sizeof(float);
  const size_t sh = (size_t)OPT_HS_POS * NS * NT * sizeof(float);   // h of one 16-position sub-tile
  return 1024 + nst * stage + bct + sh + 256;
}

// DET: the sums across warps and CTAs go to the partials of the deterministic build (see ScanBwdTmaParams), not to atomics
template <typename T, int NP, int MODE, bool DET>
__device__ __forceinline__ void scan_op_bwd_tma_body(const ScanBwdTmaParams &p) {
  constexpr int LT = OpT<T>::LT, PITCH = 2 * NP + 4, G = 4, SUB = OPT_HS_POS, GPS = SUB / G;   // 4 groups per sub-tile
  constexpr int LPC = BwdCfg<NP>::LPC, NS = BwdCfg<NP>::NS, CPW = BwdCfg<NP>::CPW;
  constexpr float kLn2 = 0.6931471805599453f;

  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char *smem = reinterpret_cast<unsigned char *>(((uintptr_t)smem_dyn + 1023) & ~(uintptr_t)1023);
  const int DT = p.DT, NST = p.nst, NT = DT * LPC;
  const int u_b = DT * OPT_ROW_BYTES, bc_b = NP * OPT_ROW_BYTES, stage_b = 3 * u_b + 2 * bc_b;
  float *bct_all = reinterpret_cast<float *>(smem + (size_t)NST * stage_b);
  float4 *sH = reinterpret_cast<float4 *>(bct_all + (NT / 32) * LT * PITCH);   // [position][state quad][thread]
  uint64_t *full = reinterpret_cast<uint64_t *>(sH + (size_t)OPT_HS_POS * (NS / 4) * NT);
  uint32_t *done = reinterpret_cast<uint32_t *>(full + NST);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = NT >> 5;
  const int half = lane / CPW, cl = lane - half * CPW;
  const int row = warp * CPW + cl;                 // this thread's channel row inside the CTA's tiles
  const int n0 = half * NS;                        // first state of this lane
  const int g = blockIdx.x / p.ctiles_per_group, ct = blockIdx.x - g * p.ctiles_per_group;
  const int d0 = g * p.dpg + ct * DT, d = d0 + row;
  const int b = blockIdx.z, split = blockIdx.y;
  const int t0 = split * p.tiles_per_split, t1 = min(p.ntiles, t0 + p.tiles_per_split);

  if (tid == 0) {
    for (int s = 0; s < NST; ++s) { mbar_init(&full[s], 1); done[s] = 0; }
    fence_mbar_init();
  }
  __syncthreads();
  if (t0 >= t1) {
    if (DET) {   // an empty segment's partials are zero
      const long long seg = (long long)b * p.nsplit + split;
#pragma unroll
      for (int s = 0; s < NS; ++s) p.part_dA[(seg * p.dim + d) * p.N + n0 + s] = 0.f;
      if (half == 0) {
        if (p.dD) p.part_dD[seg * p.dim + d] = 0.f;
        if (p.dbias) p.part_db[seg * p.dim + d] = 0.f;
      }
    }
    return;
  }

  // tiles are walked from t1-1 down to t0; k = t1-1-tau is the ring order
  auto request_tile = [&](int k, int st) {
    unsigned char *dst = smem + (size_t)st * stage_b;
    const int l0 = (t1 - 1 - k) * LT;
    mbar_arrive_expect_tx(&full[st], (uint32_t)stage_b);
    tma_load_3d(dst, &p.m_u, &full[st], l0, d0, b);
    tma_load_3d(dst + u_b, &p.m_dl, &full[st], l0, d0, b);
    tma_load_3d(dst + 2 * u_b, &p.m_do, &full[st], l0, d0, b);
    tma_load_4d(dst + 3 * u_b, &p.m_B, &full[st], l0, 0, g, b);
    tma_load_4d(dst + 3 * u_b + bc_b, &p.m_C, &full[st], l0, 0, g, b);
  };
  const int ntl = t1 - t0;
  if (tid == 0) {
    tma_prefetch_desc(&p.m_u); tma_prefetch_desc(&p.m_dl); tma_prefetch_desc(&p.m_do);
    tma_prefetch_desc(&p.m_B); tma_prefetch_desc(&p.m_C); tma_prefetch_desc(&p.m_du); tma_prefetch_desc(&p.m_dd);
    for (int k = 0; k < min(ntl, NST); ++k) request_tile(k, k);
  }

  float a2[NS], dh[NS], dAacc[NS];
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    a2[s] = p.A[(long long)d * p.N + n0 + s] * kLog2e;
    dh[s] = 0.f;
    dAacc[s] = 0.f;
  }
  if (MODE == MODE_APPLY) {
    const float *cr = p.carry + (((long long)b * p.dim + d) * p.nsplit + split) * 2 * NP + NP + n0;
#pragma unroll
    for (int s = 0; s < NS; ++s) dh[s] = cr[s];
  }
  const float bias = p.bias ? p.bias[d] : 0.f;
  const float Dv = p.D ? p.D[d] : 0.f;
  const bool sp = p.softplus != 0;
  float dDacc = 0.f, dbacc = 0.f;
  float *bct = bct_all + warp * LT * PITCH;
  float4 *sHt = sH + tid;
  float *dBg = p.dB + ((long long)b * p.G + g) * p.N * (long long)p.L;
  float *dCg = p.dC + ((long long)b * p.G + g) * p.N * (long long)p.L;

  int st = 0, ph = 0;
  for (int k = 0; k < ntl; ++k) {
    const int tau = t1 - 1 - k;
    mbar_spin(&full[st], (uint32_t)ph);
    unsigned char *sU = smem + (size_t)st * stage_b;
    unsigned char *sDl = sU + u_b;
    const unsigned char *sDo = sU + 2 * u_b;
    __syncwarp();
    transpose_bc<T, NP>(sU + 3 * u_b, sU + 3 * u_b + bc_b, bct, lane);
    __syncwarp();
    const int npos = min(LT, p.L - tau * LT);
    const int ngt = (npos + G - 1) / G;      // L is a multiple of 4 positions on this path: groups are whole
    // sub-tiles of 16 positions (fp32: the tile; 16-bit: two per tile), last first; each has its own start state in hs
#pragma unroll 1
    for (int sub = (ngt - 1) / GPS; sub >= 0; --sub) {
    const int gbase = sub * GPS, ng = min(GPS, ngt - gbase);

    // ---- forward inside the tile from its start state, h after every position -> shared memory ----
    {
      float h[NS];
      const float4 *hrow = reinterpret_cast<const float4 *>(p.hs + (((long long)b * p.dim + d) * p.nhs + (tau * LT) / SUB + sub) * NP + n0);
#pragma unroll
      for (int q = 0; q < NS / 4; ++q) { const float4 v = hrow[q]; h[4 * q] = v.x; h[4 * q + 1] = v.y; h[4 * q + 2] = v.z; h[4 * q + 3] = v.w; }
#pragma unroll 1
      for (int gi = 0; gi < ng; ++gi) {
        float raw[G], uu[G];
        load_group<T, G>(sDl, row, gbase + gi, raw);
        load_group<T, G>(sU, row, gbase + gi, uu);
#pragma unroll
        for (int i = 0; i < G; ++i) {
          const float r = raw[i] + bias;
          const float dl = sp ? softplus20(r) : r;
          const float du = dl * uu[i];
          const float *brow = bct + ((gbase + gi) * G + i) * PITCH + n0;
#pragma unroll
          for (int q = 0; q < NS / 4; ++q) {
            const float4 bv = *reinterpret_cast<const float4 *>(brow + 4 * q);
            const f2 a01 = mul2(f2{dl, dl}, f2{a2[4 * q], a2[4 * q + 1]});
            const f2 a23 = mul2(f2{dl, dl}, f2{a2[4 * q + 2], a2[4 * q + 3]});
            const f2 h01 = fma2(f2{ex2(a01.x), ex2(a01.y)}, f2{h[4 * q], h[4 * q + 1]}, mul2(f2{du, du}, f2{bv.x, bv.y}));
            const f2 h23 = fma2(f2{ex2(a23.x), ex2(a23.y)}, f2{h[4 * q + 2], h[4 * q + 3]}, mul2(f2{du, du}, f2{bv.z, bv.w}));
            h[4 * q] = h01.x; h[4 * q + 1] = h01.y; h[4 * q + 2] = h23.x; h[4 * q + 3] = h23.y;
            sHt[((gi * G + i) * (NS / 4) + q) * NT] = make_float4(h01.x, h01.y, h23.x, h23.y);
          }
        }
      }
    }

    // ---- reverse recurrence, groups of 4 positions from the end of the sub-tile ----
    float dAt[NS];   // dA of this sub-tile, folded into the running total below (two-level summation over L)
#pragma unroll
    for (int s = 0; s < NS; ++s) dAt[s] = 0.f;
#pragma unroll 1
    for (int gi = ng - 1; gi >= 0; --gi) {
      float raw[G], uu[G], dy[G];
      load_group<T, G>(sDl, row, gbase + gi, raw);
      load_group<T, G>(sU, row, gbase + gi, uu);
      load_group<T, G>(sDo, row, gbase + gi, dy);
      float rB[G], rC[G], duv[G], ddv[G];
      int which = 0;
#pragma unroll
      for (int ii = 0; ii < G; ++ii) {
        const int i = G - 1 - ii;
        const float r = raw[i] + bias;
        const float dl = sp ? softplus20(r) : r;
        const float dlu = dl * uu[i];
        const float *brow = bct + ((gbase + gi) * G + i) * PITCH + n0;
        float cB[NS], cC[NS];
        f2 s1 = f2{0.f, 0.f}, s2 = f2{0.f, 0.f};   // Σ dh·B and Σ t·a2 over this lane's states
#pragma unroll
        for (int q = 0; q < NS / 4; ++q) {
          const float4 bv = *reinterpret_cast<const float4 *>(brow + 4 * q);
          const float4 cv = *reinterpret_cast<const float4 *>(brow + NP + 4 * q);
          const float4 hv = sHt[((gi * G + i) * (NS / 4) + q) * NT];
#pragma unroll
          for (int hp = 0; hp < 2; ++hp) {
            const int s = 4 * q + 2 * hp;
            const f2 Bp = hp == 0 ? f2{bv.x, bv.y} : f2{bv.z, bv.w};
            const f2 Cp = hp == 0 ? f2{cv.x, cv.y} : f2{cv.z, cv.w};
            const f2 hp2 = hp == 0 ? f2{hv.x, hv.y} : f2{hv.z, hv.w};
            const f2 arg = mul2(f2{dl, dl}, f2{a2[s], a2[s + 1]});
            const f2 a = f2{ex2(arg.x), ex2(arg.y)};
            const f2 dhn = fma2(f2{dy[i], dy[i]}, Cp, f2{dh[s], dh[s + 1]});   // gradient reaching h_i (bwd_kernel.cuh:173-199)
            const f2 cc = mul2(f2{dy[i], dy[i]}, hp2);                         // dC term (:225)
            const f2 ahp = fma2(f2{-dlu, -dlu}, Bp, hp2);                      // a·h_{i-1} = h_i - delta·u·B
            const f2 t = mul2(dhn, ahp);
            s1 = fma2(dhn, Bp, s1);
            s2 = fma2(t, f2{a2[s], a2[s + 1]}, s2);
            const f2 da = fma2(t, f2{dl, dl}, f2{dAt[s], dAt[s + 1]});         // (:208)
            dAt[s] = da.x; dAt[s + 1] = da.y;
            const f2 cb = mul2(dhn, f2{dlu, dlu});                             // dB term (:224)
            const f2 dhm = mul2(dhn, a);
            dh[s] = dhm.x; dh[s + 1] = dhm.y;
            cB[s] = cb.x; cB[s + 1] = cb.y; cC[s] = cc.x; cC[s + 1] = cc.y;
          }
        }
        // dB / dC: sum over the CPW channels of this warp that share the lane's state set
        int wb = 0, wc = 0;
        rB[i] = transpose_reduce<NS, CPW / 2>(cB, lane, wb);
        rC[i] = transpose_reduce<NS, CPW / 2>(cC, lane, wc);
        which = wb;
        float sdhB = s1.x + s1.y, stA = s2.x + s2.y;
        if (LPC == 2) {
          sdhB += __shfl_xor_sync(0xffffffffu, sdhB, 16);
          stA += __shfl_xor_sync(0xffffffffu, stA, 16);
        }
        float ddl = fmaf(uu[i], sdhB, stA * kLn2);                            // (:206)
        duv[i] = fmaf(dy[i], Dv, dl * sdhB);                                  // (:205, :143, :250)
        dDacc = fmaf(dy[i], uu[i], dDacc);                                    // (:144)
        if (sp && r <= 20.f) ddl *= __fdividef(1.f, 1.f + ex2(-r * kLog2e));  // (:241-245)
        dbacc += ddl;
        ddv[i] = ddl;
      }
      if (half == 0) {
        store_group<T, G>(sU, row, gbase + gi, duv);     // du over u, ddelta over delta: in place
        store_group<T, G>(sDl, row, gbase + gi, ddv);
      }
      // one vector atomic per state and 4 positions; the value index `which` is held by CPW / NS lanes: the lowest issues
      constexpr int DUP = CPW / NS;
      if ((cl & (DUP - 1)) == 0) {
        const long long off = (long long)(n0 + which) * p.L + (long long)tau * LT + (gbase + gi) * G;
        if (DET) {
          const long long tile = (long long)ct * nwarps + warp;
          const long long po = (tile * p.batch * p.G + (long long)b * p.G + g) * p.N * (long long)p.L + off;
          *reinterpret_cast<float4 *>(p.part_B + po) = make_float4(rB[0], rB[1], rB[2], rB[3]);
          *reinterpret_cast<float4 *>(p.part_C + po) = make_float4(rC[0], rC[1], rC[2], rC[3]);
        } else {
          red_add_v4(dBg + off, rB[0], rB[1], rB[2], rB[3]);
          red_add_v4(dCg + off, rC[0], rC[1], rC[2], rC[3]);
        }
      }
    }
#pragma unroll
    for (int s = 0; s < NS; ++s) dAacc[s] += dAt[s];
    }   // sub-tiles

    // this warp's rows of du / ddelta -> global; the slot may be refilled once the stores have READ it (a tile of the
    // backward is ~4x the forward's work, so the wait is small against it and the ring stays at 2 stages)
    fence_proxy_async();
    __syncwarp();
    if (lane == 0) {
      tma_store_3d(&p.m_du, sU + warp * CPW * OPT_ROW_BYTES, tau * LT, d0 + warp * CPW, b);
      tma_store_3d(&p.m_dd, sDl + warp * CPW * OPT_ROW_BYTES, tau * LT, d0 + warp * CPW, b);
      tma_store_commit();
      tma_store_wait_read<0>();
      if (k + NST < ntl) {
        const uint32_t old = smem_inc_acq_rel(&done[st]);
        if ((old + 1) % (uint32_t)nwarps == 0) request_tile(k + NST, st);
      }
    }
    __syncwarp();
    if (++st == NST) { st = 0; ph ^= 1; }
  }
  if (lane == 0) tma_store_wait_all<0>();

  if (DET) {
    const long long seg = (long long)b * p.nsplit + split;
#pragma unroll
    for (int s = 0; s < NS; ++s) p.part_dA[(seg * p.dim + d) * p.N + n0 + s] = dAacc[s];
    if (half == 0) {
      if (p.dD) p.part_dD[seg * p.dim + d] = dDacc;
      if (p.dbias) p.part_db[seg * p.dim + d] = dbacc;
    }
    return;
  }
#pragma unroll
  for (int s = 0; s < NS; ++s) atomicAdd(&p.dA[(long long)d * p.N + n0 + s], dAacc[s]);   // over batch and segments (:262-273)
  if (half == 0) {
    if (p.dD) atomicAdd(&p.dD[d], dDacc);
    if (p.dbias) atomicAdd(&p.dbias[d], dbacc);
  }
}

template <typename T, int NP, int MODE>
__global__ void __launch_bounds__(128, 2) scan_op_bwd_tma_kernel(const __grid_constant__ ScanBwdTmaParams p) {
  scan_op_bwd_tma_body<T, NP, MODE, false>(p);
}

template <typename T, int NP, int MODE>
__global__ void __launch_bounds__(128, 2) scan_op_bwd_tma_det_kernel(const __grid_constant__ ScanBwdTmaParams p) {
  scan_op_bwd_tma_body<T, NP, MODE, true>(p);
}

// Reverse summary of one L-segment: P[n] = prod a over the segment, g[n] = value the reverse recurrence
// dh <- (dh + dout·C)·a hands to the position BEFORE the segment when it starts from 0 at the segment's end.
// One thread = one channel, all states (as the forward).  Loads delta, dout and C only.
template <typename T, int NP>
__global__ void __launch_bounds__(128, 4) scan_op_rev_summary_kernel(const __grid_constant__ ScanBwdTmaParams p) {
  constexpr int LT = OpT<T>::LT, PITCH = 2 * NP + 4, G = 4;
  extern __shared__ __align__(1024) unsigned char smem_dyn[];
  unsigned char *smem = reinterpret_cast<unsigned char *>(((uintptr_t)smem_dyn + 1023) & ~(uintptr_t)1023);
  const int DT = p.DT, NST = p.nst;
  const int u_b = DT * OPT_ROW_BYTES, bc_b = NP * OPT_ROW_BYTES, stage_b = 2 * u_b + 2 * bc_b;
  float *bct_all = reinterpret_cast<float *>(smem + (size_t)NST * stage_b);
  uint64_t *full = reinterpret_cast<uint64_t *>(bct_all + (DT / 32) * LT * PITCH);
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
  const int ntl = max(t1 - t0, 0);
  auto request_tile = [&](int k, int st) {
    unsigned char *dst = smem + (size_t)st * stage_b;
    const int l0 = (t1 - 1 - k) * LT;
    mbar_arrive_expect_tx(&full[st], (uint32_t)(2 * u_b + 2 * bc_b));
    tma_load_3d(dst, &p.m_dl, &full[st], l0, d0, b);
    tma_load_3d(dst + u_b, &p.m_do, &full[st], l0, d0, b);
    tma_load_4d(dst + 2 * u_b, &p.m_C, &full[st], l0, 0, g, b);          // transpose_bc takes two raw tiles: C twice
    tma_load_4d(dst + 2 * u_b + bc_b, &p.m_C, &full[st], l0, 0, g, b);
  };
  if (tid == 0) for (int k = 0; k < min(ntl, NST); ++k) request_tile(k, k);

  float a2[NP], gsum[NP];
#pragma unroll
  for (int s = 0; s < NP; ++s) { a2[s] = p.A[(long long)d * p.N + s] * kLog2e; gsum[s] = 0.f; }
  const float bias = p.bias ? p.bias[d] : 0.f;
  const bool sp = p.softplus != 0;
  float sumdl = 0.f;
  float *bct = bct_all + warp * LT * PITCH;
  int st = 0, ph = 0;
  for (int k = 0; k < ntl; ++k) {
    const int tau = t1 - 1 - k;
    mbar_spin(&full[st], (uint32_t)ph);
    const unsigned char *sDl = smem + (size_t)st * stage_b;
    const unsigned char *sDo = sDl + u_b;
    __syncwarp();
    transpose_bc<T, NP>(sDl + 2 * u_b, sDl + 2 * u_b + bc_b, bct, lane);
    __syncwarp();
    const int npos = min(LT, p.L - tau * LT);
    const int ng = (npos + G - 1) / G;
#pragma unroll 1
    for (int gi = ng - 1; gi >= 0; --gi) {
      float raw[G], dy[G];
      load_group<T, G>(sDl, tid, gi, raw);
      load_group<T, G>(sDo, tid, gi, dy);
#pragma unroll
      for (int ii = 0; ii < G; ++ii) {
        const int i = G - 1 - ii;
        if (gi * G + i < npos) {
          const float r = raw[i] + bias;
          const float dl = sp ? softplus20(r) : r;
          const float *crow = bct + (gi * G + i) * PITCH + NP;
#pragma unroll
          for (int q = 0; q < NP / 4; ++q) {
            const float4 cv = *reinterpret_cast<const float4 *>(crow + 4 * q);
            const f2 a01 = mul2(f2{dl, dl}, f2{a2[4 * q], a2[4 * q + 1]});
            const f2 a23 = mul2(f2{dl, dl}, f2{a2[4 * q + 2], a2[4 * q + 3]});
            const f2 g01 = mul2(fma2(f2{dy[i], dy[i]}, f2{cv.x, cv.y}, f2{gsum[4 * q], gsum[4 * q + 1]}), f2{ex2(a01.x), ex2(a01.y)});
            const f2 g23 = mul2(fma2(f2{dy[i], dy[i]}, f2{cv.z, cv.w}, f2{gsum[4 * q + 2], gsum[4 * q + 3]}), f2{ex2(a23.x), ex2(a23.y)});
            gsum[4 * q] = g01.x; gsum[4 * q + 1] = g01.y; gsum[4 * q + 2] = g23.x; gsum[4 * q + 3] = g23.y;
          }
          sumdl += dl;
        }
      }
    }
    __syncwarp();
    if (lane == 0 && k + NST < ntl) {
      const uint32_t old = smem_inc_acq_rel(&done[st]);
      if ((old + 1) % (uint32_t)nwarps == 0) request_tile(k + NST, st);
    }
    if (++st == NST) { st = 0; ph ^= 1; }
  }
  float *cr = p.carry + (((long long)b * p.dim + d) * p.nsplit + split) * 2 * NP;
#pragma unroll
  for (int s = 0; s < NP; ++s) { cr[s] = ex2(a2[s] * sumdl); cr[NP + s] = gsum[s]; }
}

// carry[row][split] = (P, g_local) -> (., dh entering the segment from its right neighbour): chained from the LAST segment
__global__ void scan_combine_rev_kernel(float *carry, long long nrows, int nsplit, int NP) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nrows * NP) return;
  const long long row = idx / NP;
  const int n = (int)(idx - row * NP);
  float Hc = 0.f;
  float *base = carry + row * nsplit * 2 * NP + n;
  for (int s0 = nsplit - 1; s0 >= 0; s0 -= 8) {      // eight segments per round: their loads are issued together (see scan_combine_kernel)
    float P[8], gl[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool in = s0 - j >= 0;
      P[j] = in ? base[(long long)(s0 - j) * 2 * NP] : 1.f;
      gl[j] = in ? base[(long long)(s0 - j) * 2 * NP + NP] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (s0 - j >= 0) {
        base[(long long)(s0 - j) * 2 * NP + NP] = Hc;
        Hc = fmaf(P[j], Hc, gl[j]);
      }
    }
  }
}

// ---- host side ----
constexpr int kBwdMaxSplit = 64;

// scratch of the deterministic build: [dB partials] [dC partials] (dpg / CPW, batch, G, N, L) [dA partials (batch·64, dim, N)]
// [dD partials] [ddelta_bias partials] (batch·64, dim)
size_t scan_op_bwd_tma_det_bytes(int batch, int dim, int L, int N, int G) {
  const size_t cpw = N >= 16 ? 16 : 32, ntile = (size_t)(dim / G) / cpw, segs = (size_t)batch * kBwdMaxSplit;
  return 2 * align256(ntile * batch * G * N * L * sizeof(float)) + align256(segs * dim * N * sizeof(float)) + 2 * align256(segs * dim * sizeof(float));
}

// workspace = [hs (batch, dim, ntiles, N)] [forward-split carry] [reverse-split carry]
size_t scan_op_bwd_tma_workspace_bytes(int batch, int dim, int L, int N, int elem_bytes) {
  (void)elem_bytes;
  const size_t nhs = (L + OPT_HS_POS - 1) / OPT_HS_POS;
  return align256((size_t)batch * dim * nhs * N * sizeof(float)) + align256(scan_op_tma_workspace_bytes(batch, dim, N)) +
         align256((size_t)batch * dim * kBwdMaxSplit * 2 * N * sizeof(float));
}

template <typename T>
static ScanOpPlan bwd_tma_plan(int batch, int dim, int L, int N, int G, int force_split) {
  constexpr int LT = OpT<T>::LT;
  const int NP = N, dpg = dim / G;
  ScanOpPlan pl;
  pl.DT = (dpg % 64 == 0) ? 64 : 32;
  pl.ntiles = (L + LT - 1) / LT;
  // L-segments: the reverse summaries are a cheap extra sweep (no h, no reductions: ~0.3 of the main sweep), so fill whole
  // waves of the resident CTA slots (2 x 128-thread CTAs per SM at d_state 16, ~5 x 64-thread CTAs below)
  const int lpc = NP >= 16 ? 2 : 1;
  int nsplit = pick_segments((long long)batch * G * (dpg / pl.DT), pl.ntiles, kNumSMs * (lpc == 2 ? 2 : 5), 1.3, kBwdMaxSplit);
  if (force_split > 0) nsplit = std::min(force_split, kBwdMaxSplit);
  int tps = std::max(1, (pl.ntiles + nsplit - 1) / nsplit);
  pl.tiles_per_split = tps;
  pl.nsplit = std::max(1, (pl.ntiles + tps - 1) / tps);
  {
    const size_t stage = (size_t)3 * pl.DT * OPT_ROW_BYTES + (size_t)2 * NP * OPT_ROW_BYTES;
    const size_t budget = (size_t)(227 * 1024) / (lpc == 2 ? 2 : 4) - 1024;   // 2 x 128-thread / 4 x 64-thread CTAs per SM
    size_t base;
    switch (NP) {
      case 4: base = bwd_tma_smem_bytes<T, 4>(pl.DT, 0); break;
      case 8: base = bwd_tma_smem_bytes<T, 8>(pl.DT, 0); break;
      default: base = bwd_tma_smem_bytes<T, 16>(pl.DT, 0); break;
    }
    int nst = budget > base ? (int)((budget - base) / stage) : 2;
    pl.nst = std::max(2, std::min(4, nst));
  }
  return pl;
}

// Launch plan of the main (reverse) sweep of scan_op_bwd_tma (host only; eligibility guarantees N in {4, 8, 16}).  Its state
// sweep is scan_op_fwd_tma with the same force_split and the forward-carry part of the workspace (scan_op_fwd_tma_plan).
ScanOpPlan scan_op_bwd_tma_plan(int elem_bytes, int batch, int dim, int L, int N, int G, int force_split) {
  return elem_bytes == 4 ? bwd_tma_plan<float>(batch, dim, L, N, G, force_split) : bwd_tma_plan<__half>(batch, dim, L, N, G, force_split);
}

template <typename T, int NP>
static int launch_bwd_tma(ScanBwdTmaParams &p, cudaStream_t stream) {
  constexpr int LPC = BwdCfg<NP>::LPC;
  auto prep = [&](const void *fn, size_t smem) -> cudaError_t { (void)smem; return prep_kernel_once(fn); };
  dim3 grid(p.G * p.ctiles_per_group, p.nsplit, p.batch);
  if (p.nsplit > 1) {
    const size_t smem = 1024 + (size_t)p.nst * (2 * p.DT * OPT_ROW_BYTES + 2 * NP * OPT_ROW_BYTES) +
                        (size_t)(p.DT / 32) * OpT<T>::LT * (2 * NP + 4) * sizeof(float) + 256;
    auto ks = scan_op_rev_summary_kernel<T, NP>;
    SIGMA_CHECK_CUDA(prep((const void *)ks, smem));
    ks<<<grid, p.DT, smem, stream>>>(p);
    SIGMA_CHECK_LAUNCH();
    const long long nrows = (long long)p.batch * p.dim, tot = nrows * NP;
    scan_combine_rev_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(p.carry, nrows, p.nsplit, NP);
    SIGMA_CHECK_LAUNCH();
  }
  const size_t smem = bwd_tma_smem_bytes<T, NP>(p.DT, p.nst);
  const bool det = p.part_B != nullptr;
  auto k = p.nsplit == 1 ? (det ? scan_op_bwd_tma_det_kernel<T, NP, MODE_SERIAL> : scan_op_bwd_tma_kernel<T, NP, MODE_SERIAL>)
                         : (det ? scan_op_bwd_tma_det_kernel<T, NP, MODE_APPLY> : scan_op_bwd_tma_kernel<T, NP, MODE_APPLY>);
  SIGMA_CHECK_CUDA(prep((const void *)k, smem));
  k<<<grid, p.DT * LPC, smem, stream>>>(p);
  SIGMA_CHECK_LAUNCH();
  if (!det) return SIGMA_OK;
  // fixed-order sums: dB / dC over the warp channel tiles of a group, dA / dD / ddelta_bias over (batch, segment)
  const int ntile = p.dpg / BwdCfg<NP>::CPW, segs = p.batch * p.nsplit;
  const long long bgnl = (long long)p.batch * p.G * p.N * p.L, dn = (long long)p.dim * p.N;
  int rc;
  if ((rc = sum_parts_det_launch(p.part_B, ntile, bgnl, bgnl, 0, p.dB, stream))) return rc;
  if ((rc = sum_parts_det_launch(p.part_C, ntile, bgnl, bgnl, 0, p.dC, stream))) return rc;
  if ((rc = sum_parts_det_launch(p.part_dA, segs, dn, dn, 0, p.dA, stream))) return rc;
  if (p.dD && (rc = sum_parts_det_launch(p.part_dD, segs, p.dim, p.dim, 0, p.dD, stream))) return rc;
  if (p.dbias && (rc = sum_parts_det_launch(p.part_db, segs, p.dim, p.dim, 0, p.dbias, stream))) return rc;
  return SIGMA_OK;
}

// All tensors contiguous, element type T (dB / dC / dA / dD / dbias fp32, OVERWRITTEN).  Caller checked eligibility
// (scan_op_tma_eligible) with contiguous strides.
template <typename T>
int scan_op_bwd_tma(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                    const float *bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC, float *dD,
                    float *dbias, int batch, int dim, int L, int N, int G, int softplus, void *ws, size_t ws_bytes,
                    int force_split, cudaStream_t stream, void *det_ws) {
  constexpr int LT = OpT<T>::LT;
  const int NP = N;
  if (ws == nullptr || ws_bytes < scan_op_bwd_tma_workspace_bytes(batch, dim, L, N, (int)sizeof(T))) {
    set_error("sigma_scan_bwd: workspace too small (%zu < %zu)", ws_bytes, scan_op_bwd_tma_workspace_bytes(batch, dim, L, N, (int)sizeof(T)));
    return SIGMA_EWORKSPACE;
  }
  const int ntiles = (L + LT - 1) / LT;
  const size_t hs_b = align256((size_t)batch * dim * ((L + OPT_HS_POS - 1) / OPT_HS_POS) * N * sizeof(float));
  const size_t fc_b = align256(scan_op_tma_workspace_bytes(batch, dim, N));
  float *hs = (float *)ws;
  void *fcarry = (char *)ws + hs_b;
  float *rcarry = (float *)((char *)ws + hs_b + fc_b);

  sigma_scan_strides st;
  st.u_batch = st.delta_batch = st.out_batch = (int64_t)dim * L;
  st.u_dim = st.delta_dim = st.out_dim = L;
  st.A_dim = N; st.A_dstate = 1;
  st.B_batch = st.C_batch = (int64_t)G * N * L;
  st.B_group = st.C_group = (int64_t)N * L;
  st.B_dstate = st.C_dstate = L;
  // 1. state sweep (no y): hs
  int rc = scan_op_fwd_tma<T>(u, delta, A, B, C, D, bias, nullptr, nullptr, hs, batch, dim, L, N, G, softplus, st, fcarry, fc_b,
                              force_split, stream);
  if (rc) return rc;

  SIGMA_CHECK_CUDA(cudaMemsetAsync(dA, 0, (size_t)dim * N * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dB, 0, (size_t)batch * G * N * L * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dC, 0, (size_t)batch * G * N * L * sizeof(float), stream));
  if (dD) SIGMA_CHECK_CUDA(cudaMemsetAsync(dD, 0, (size_t)dim * sizeof(float), stream));
  if (dbias) SIGMA_CHECK_CUDA(cudaMemsetAsync(dbias, 0, (size_t)dim * sizeof(float), stream));

  ScanBwdTmaParams p;
  memset(&p, 0, sizeof(p));
  p.A = A; p.D = D; p.bias = bias; p.hs = hs;
  p.dA = dA; p.dB = dB; p.dC = dC; p.dD = dD; p.dbias = dbias; p.carry = rcarry;
  p.batch = batch; p.dim = dim; p.L = L; p.N = N; p.G = G; p.dpg = dim / G; p.softplus = softplus;
  if (det_ws) {   // layout of scan_op_bwd_tma_det_bytes
    const size_t cpw = N >= 16 ? 16 : 32, ntile = (size_t)p.dpg / cpw, segs = (size_t)batch * kBwdMaxSplit;
    const size_t bc = align256(ntile * batch * G * N * L * sizeof(float)), da = align256(segs * dim * N * sizeof(float));
    const size_t dd = align256(segs * dim * sizeof(float));
    char *w = (char *)det_ws;
    p.part_B = (float *)w; p.part_C = (float *)(w + bc); p.part_dA = (float *)(w + 2 * bc);
    p.part_dD = (float *)(w + 2 * bc + da); p.part_db = (float *)(w + 2 * bc + da + dd);
  }
  const ScanOpPlan pl = scan_op_bwd_tma_plan((int)sizeof(T), batch, dim, L, N, G, force_split);
  p.DT = pl.DT;
  p.ctiles_per_group = p.dpg / p.DT;
  p.ntiles = ntiles;
  p.nhs = (L + OPT_HS_POS - 1) / OPT_HS_POS;
  p.tiles_per_split = pl.tiles_per_split;
  p.nsplit = pl.nsplit;
  p.nst = pl.nst;
  const int lpc = NP >= 16 ? 2 : 1;   // lanes per channel (BwdCfg)
  const uint64_t sz = sizeof(T);
  {
    uint64_t dims[3] = {(uint64_t)L, (uint64_t)dim, (uint64_t)batch};
    uint64_t str[2] = {(uint64_t)L * sz, (uint64_t)dim * L * sz};
    uint32_t box[3] = {(uint32_t)LT, (uint32_t)p.DT, 1};
    uint32_t boxw[3] = {(uint32_t)LT, (uint32_t)(32 / lpc), 1};
    const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_64B;
    if ((rc = make_tmap(&p.m_u, OpT<T>::kType, 3, u, dims, str, box, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if ((rc = make_tmap(&p.m_dl, OpT<T>::kType, 3, delta, dims, str, box, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if ((rc = make_tmap(&p.m_do, OpT<T>::kType, 3, dout, dims, str, box, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if ((rc = make_tmap(&p.m_du, OpT<T>::kType, 3, du, dims, str, boxw, sw, CU_TENSOR_MAP_L2_PROMOTION_NONE))) return rc;
    if ((rc = make_tmap(&p.m_dd, OpT<T>::kType, 3, ddelta, dims, str, boxw, sw, CU_TENSOR_MAP_L2_PROMOTION_NONE))) return rc;
    uint64_t dimb[4] = {(uint64_t)L, (uint64_t)N, (uint64_t)G, (uint64_t)batch};
    uint64_t strb[3] = {(uint64_t)L * sz, (uint64_t)N * L * sz, (uint64_t)G * N * L * sz};
    uint32_t boxb[4] = {(uint32_t)LT, (uint32_t)NP, 1, 1};
    if ((rc = make_tmap(&p.m_B, OpT<T>::kType, 4, B, dimb, strb, boxb, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
    if ((rc = make_tmap(&p.m_C, OpT<T>::kType, 4, C, dimb, strb, boxb, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B))) return rc;
  }
  switch (NP) {
    case 4: return launch_bwd_tma<T, 4>(p, stream);
    case 8: return launch_bwd_tma<T, 8>(p, stream);
    default: return launch_bwd_tma<T, 16>(p, stream);
  }
}

#define SIGMA_INST(T)                                                                                                         \
  template int scan_op_bwd_tma<T>(const void *, const void *, const float *, const void *, const void *, const float *,       \
                                  const float *, const void *, void *, void *, float *, float *, float *, float *, float *,   \
                                  int, int, int, int, int, int, void *, size_t, int, cudaStream_t, void *);
SIGMA_INST(float)
SIGMA_INST(__half)
SIGMA_INST(__nv_bfloat16)
#undef SIGMA_INST

}  // namespace sigma
