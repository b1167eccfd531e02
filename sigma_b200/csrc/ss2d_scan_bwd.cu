// f1 — backward of the FUSED multi-direction SS2D scan, channels-last (see include/sigma_b200.h: sigma_ss2d_scan_bwd_saved).
//
// Replaces, for training, the autograd of CrossScan + dt_proj einsum + SelectiveScan + CrossMerge
// (vmamba.py:80-121, 195-215 and selective_scan_bwd_kernel.cuh:68-274) without ever materialising CrossScan's (B,4,D,L)
// copy: every direction is the same 4-D TMA walk over the channels-last tensors that the forward uses.  The training forward
// (sigma_ss2d_scan_fwd_save) has already written delta' = softplus(dt_r·W_dt + bias) -> `delta` slabs (K,B,L,D), and the state
// h at the start of every 16-position tile -> `hs`; both are inputs here.  Two sweeps:
//   1. reverse summaries (ss2d_bwd_kernel<MODE_SUMMARY>, only with L-segments) + scan_combine_rev_kernel: the dh entering
//      every segment (L-parallel reverse sweep);
//   2. main sweep (ss2d_bwd_kernel, tiles walked BACKWARDS): per tile recompute h at every position from the tile's start
//      state into shared memory, then the reverse recurrence dh_l = a_{l+1}·dh_{l+1} + dy_l·C_l producing
//        du      -> TMA REDUCE-ADD (cp.reduce.async.bulk.tensor .add.f32) straight into dxc (B,L,D): the four directions'
//                   contributions meet in L2, no (B,4,D,L) gradient tensor and no CrossScan backward;
//        ddelta  -> `ddelta` slabs (K,B,L,D) (pre-softplus; the caller turns them into d dt_r and dW_dt with two GEMMs);
//        dB, dC  -> summed over the warp's channels by the transposing shuffle reduction of the op-level backward, then
//                   coalesced red.global.add into dxdbl (B,L,K,Cp);
//        dA, dDs, d dt_bias -> per-thread accumulators, one atomic per channel at the end.
// Thread mapping as scan_op_bwd_tma.cu: d_state 16 -> 2 lanes per channel (8 states each), d_state 4 -> 1; a CTA = 64
// channels of one (direction, image [, L-segment]); tiles of 16 positions through a TMA ring (full mbarrier + last-arriver
// refill).  Kinds SIGMA_DIRS_CROSS4 and SIGMA_DIRS_SEQ2 (SS2D and ConMB) and SIGMA_DIRS_CROSS (CroMB: one row-major walk per
// image of a 2·images batch, per-modality weights, C from the other modality; separate *_cross_kernel instances, no
// deterministic build); d_state in {4, 16}; D % 64 == 0.
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "scan_core.cuh"
#include "tma.cuh"

namespace sigma {

constexpr int FB_LT = 16;   // positions per tile
constexpr int FB_DT = 64;   // channels per CTA

struct alignas(64) Ss2dBwdParams {
  CUtensorMap m_xc[4], m_dy[4], m_dl[4], m_dbl[4];    // loads: boxes {64 ch, 16 pos} / {Cp, 16 pos}
  CUtensorMap m_dxc[4], m_dd[4];                      // per-warp outputs: boxes {CPW ch, 16 pos}
  const float *dtw, *dtb, *A, *Ds, *hs;
  float *dxdbl, *dA, *dDs, *ddtb, *carry;
  int D, N, R, Cp, K, batch;
  long long Lseq;
  int I[4], O[4], rev[4];
  long long psi[4], pso[4];     // position = o·pso + i·psi
  int nsplit, tiles_per_split, max_tiles, nst;
  // deterministic build (ss2d_bwd_det_kernel): m_dxc points at the du slabs (K, batch, Lseq, D); dB / dC partials per warp
  // channel tile (D / CPW, batch, Lseq, K, 2N); dA (batch·nsplit, K·D, N), dDs and d dt_bias (batch·nsplit, K·D) per
  // (image, L-segment)
  float *part_bc, *part_dA, *part_dD, *part_db;
};

template <int N> struct FbCfg {
  static constexpr int LPC = N >= 16 ? 2 : 1;
  static constexpr int NS = N / LPC;
  static constexpr int CPW = 32 / LPC;
};

// everything both sweeps share: CTA coordinates, the direction's tile geometry, the ring
struct FbWalk {
  int k, split, b, d0, t0, t1, I, TPO, ntiles;
  bool rev;
  __device__ __forceinline__ void tile(int tau, int &o, int &i0, int &npos) const {
    const int tm = rev ? ntiles - 1 - tau : tau;
    o = tm / TPO;
    i0 = (tm - o * TPO) * FB_LT;
    npos = min(FB_LT, I - i0);
  }
};

__device__ __forceinline__ FbWalk fb_walk(const Ss2dBwdParams &p) {
  FbWalk w;
  w.d0 = blockIdx.x * FB_DT;
  w.k = blockIdx.y / p.nsplit;
  w.split = blockIdx.y - w.k * p.nsplit;
  w.b = blockIdx.z;
  w.I = p.I[w.k];
  w.rev = p.rev[w.k] != 0;
  w.TPO = (w.I + FB_LT - 1) / FB_LT;
  w.ntiles = p.O[w.k] * w.TPO;
  w.t0 = w.split * p.tiles_per_split;
  w.t1 = min(w.ntiles, w.t0 + p.tiles_per_split);
  return w;
}

// ---------------------------------------------------------------------------------------------------------------------
// 1 + 2. reverse summaries (MODE_SUMMARY) and the main backward sweep (MODE_SERIAL / MODE_APPLY)
// ---------------------------------------------------------------------------------------------------------------------
// DET: every sum across CTAs goes to the partials of the deterministic build (see Ss2dBwdParams) instead of an atomic.
// CROSS: image b runs with weight set kw = [b >= batch/2] and reads C from image bC = the other modality's (as the forward):
// the stage holds bC's x_dbl tile too, dC goes to the C columns of bC's dxdbl rows, dA / dDs / d dt_bias to rows kw·D + d.
// XT: element type of the xc, dy and delta' tiles (float; __nv_bfloat16 / __half in the bf16 / fp16 training modes, which widen
// them on the read from the stage and keep everything else — x_dbl, hs, every accumulator, du / ddelta and their TMA stores — fp32).
template <int N, int MODE, bool DET, bool CROSS, typename XT = float>
__device__ __forceinline__ void ss2d_bwd_body(const Ss2dBwdParams &p) {
  static_assert(!(DET && CROSS), "no deterministic build of the CROSS backward");
  static_assert(!DET || sizeof(XT) == 4, "no deterministic build of the 16-bit backwards");
  constexpr int LPC = FbCfg<N>::LPC, NS = FbCfg<N>::NS, CPW = FbCfg<N>::CPW, NT = FB_DT * LPC;
  constexpr bool MAIN = MODE != MODE_SUMMARY;
  constexpr float kLn2 = 0.6931471805599453f;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  float *smem = reinterpret_cast<float *>(smem_raw);
  const int NST = p.nst, Cp = p.Cp;
  const int xc_fl = FB_LT * FB_DT * (int)sizeof(XT) / 4, dbl_fl = FB_LT * Cp;   // tile sizes in floats (bf16 tiles: half)
  const int stage_fl = (MAIN ? 3 : 2) * xc_fl + (CROSS ? 2 : 1) * dbl_fl;   // [xc] dy dl dbl [dbl of image bC]
  float *stage_all = smem + NST * stage_fl;                        // per-warp staging: du [16][CPW], ddelta [16][CPW]
  float4 *sH = reinterpret_cast<float4 *>(stage_all + (MAIN ? (NT / 32) * 2 * FB_LT * CPW : 0));   // [16][NS/4][NT]
  uint64_t *full = reinterpret_cast<uint64_t *>(sH + (MAIN ? FB_LT * (NS / 4) * NT : 0));
  uint32_t *done = reinterpret_cast<uint32_t *>(full + NST);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = NT >> 5;
  const int half = lane / CPW, cl = lane - half * CPW, c = warp * CPW + cl, n0 = half * NS;
  const FbWalk w = fb_walk(p);
  const int d = w.d0 + c;
  const int half_b = p.batch >> 1;
  const int kw = CROSS ? (w.b >= half_b ? 1 : 0) : w.k;
  const int bC = CROSS ? (w.b >= half_b ? w.b - half_b : w.b + half_b) : w.b;
  if (tid == 0) {
    for (int s = 0; s < NST; ++s) { mbar_init(&full[s], 1); done[s] = 0; }
    fence_mbar_init();
  }
  __syncthreads();
  if (w.t0 >= w.t1) {
    if (MODE == MODE_SUMMARY) {   // empty trailing segment: identity summary
      float *cr = p.carry + ((((long long)w.b * p.K + w.k) * p.D + d) * p.nsplit + w.split) * 2 * N;
#pragma unroll
      for (int s = 0; s < NS; ++s) { cr[n0 + s] = 1.f; cr[N + n0 + s] = 0.f; }
    } else if (DET) {              // an empty segment's partials are zero
      const long long seg = (long long)w.b * p.nsplit + w.split, wd = (long long)w.k * p.D + d;
#pragma unroll
      for (int s = 0; s < NS; ++s) p.part_dA[(seg * p.K * p.D + wd) * N + n0 + s] = 0.f;
      if (half == 0) { p.part_dD[seg * p.K * p.D + wd] = 0.f; p.part_db[seg * p.K * p.D + wd] = 0.f; }
    }
    return;
  }
  const int ntl = w.t1 - w.t0;
  const uint32_t tx = (uint32_t)(stage_fl * sizeof(float));
  // ring order kk = 0.. walks tiles t1-1 down to t0
  auto request_tile = [&](int kk, int st) {
    int o, i0, npos;
    w.tile(w.t1 - 1 - kk, o, i0, npos);
    float *dst = smem + st * stage_fl;
    mbar_arrive_expect_tx(&full[st], tx);
    if (MAIN) {
      tma_load_4d(dst, &p.m_xc[w.k], &full[st], w.d0, i0, o, w.b);
      dst += xc_fl;
    }
    tma_load_4d(dst, &p.m_dy[w.k], &full[st], w.d0, i0, o, w.b);
    tma_load_4d(dst + xc_fl, &p.m_dl[w.k], &full[st], w.d0, i0, o, w.k * p.batch + w.b);
    tma_load_4d(dst + 2 * xc_fl, &p.m_dbl[w.k], &full[st], 0, i0, o, w.b);
    if (CROSS) tma_load_4d(dst + 2 * xc_fl + dbl_fl, &p.m_dbl[w.k], &full[st], 0, i0, o, bC);
  };
  if (tid == 0) for (int kk = 0; kk < min(ntl, NST); ++kk) request_tile(kk, kk);

  float a2[NS], dh[NS], dAacc[NS];
  const long long wd = (long long)kw * p.D + d;
#pragma unroll
  for (int s = 0; s < NS; ++s) { a2[s] = p.A[wd * N + n0 + s] * kLog2e; dh[s] = 0.f; dAacc[s] = 0.f; }
  float *carry_row = p.carry + ((((long long)w.b * p.K + w.k) * p.D + d) * p.nsplit + w.split) * 2 * N;
  if (MODE == MODE_APPLY) {
#pragma unroll
    for (int s = 0; s < NS; ++s) dh[s] = carry_row[N + n0 + s];
  }
  const float Dv = MAIN ? p.Ds[wd] : 0.f;
  float dDacc = 0.f, dbacc = 0.f, sumdl = 0.f;
  float *sdu = stage_all + warp * 2 * FB_LT * CPW, *sdd = sdu + FB_LT * CPW;
  float4 *sHt = sH + tid;
  float *dxrow0 = p.dxdbl + (long long)w.b * p.Lseq * p.K * Cp + (long long)w.k * Cp;   // + pos·K·Cp
  float *dxrowC = CROSS ? p.dxdbl + (long long)bC * p.Lseq * p.K * Cp + (long long)w.k * Cp : dxrow0;

  int st = 0, ph = 0;
  for (int kk = 0; kk < ntl; ++kk) {
    const int tau = w.t1 - 1 - kk;
    int o, i0, npos;
    w.tile(tau, o, i0, npos);
    mbar_spin(&full[st], (uint32_t)ph);
    const float *base = smem + st * stage_fl;
    const XT *sXC = reinterpret_cast<const XT *>(base), *sDY = reinterpret_cast<const XT *>(base + (MAIN ? xc_fl : 0));
    const XT *sDL = reinterpret_cast<const XT *>(base + (MAIN ? 2 : 1) * xc_fl);
    const float *sDB = base + (MAIN ? 3 : 2) * xc_fl;
    const float *sDC = CROSS ? sDB + dbl_fl : sDB;   // the x_dbl tile C is read from

    if (MAIN) {
      // ---- forward inside the tile from its start state (walk order), h after every step -> shared memory ----
      float h[NS];
      const float4 *hp = reinterpret_cast<const float4 *>(p.hs +(((((long long)w.k * p.batch + w.b) * p.max_tiles + tau) * p.D + d) * N + n0));
#pragma unroll
      for (int q = 0; q < NS / 4; ++q) { const float4 v = hp[q]; h[4 * q] = v.x; h[4 * q + 1] = v.y; h[4 * q + 2] = v.z; h[4 * q + 3] = v.w; }
#pragma unroll 1
      for (int s = 0; s < npos; ++s) {
        const int r = w.rev ? npos - 1 - s : s;
        const float dl = to_f32(sDL[r * FB_DT + c]);
        const float du = dl * to_f32(sXC[r * FB_DT + c]);
        const float *row = sDB + r * Cp + n0;
#pragma unroll
        for (int q = 0; q < NS / 4; ++q) {
          const float4 bv = *reinterpret_cast<const float4 *>(row + 4 * q);
          h[4 * q] = fmaf(ex2(dl * a2[4 * q]), h[4 * q], du * bv.x);
          h[4 * q + 1] = fmaf(ex2(dl * a2[4 * q + 1]), h[4 * q + 1], du * bv.y);
          h[4 * q + 2] = fmaf(ex2(dl * a2[4 * q + 2]), h[4 * q + 2], du * bv.z);
          h[4 * q + 3] = fmaf(ex2(dl * a2[4 * q + 3]), h[4 * q + 3], du * bv.w);
          sHt[(s * (NS / 4) + q) * NT] = make_float4(h[4 * q], h[4 * q + 1], h[4 * q + 2], h[4 * q + 3]);
        }
      }
    }

    // ---- reverse recurrence over the tile's steps ----
    float dAt[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) dAt[s] = 0.f;
#pragma unroll 1
    for (int s = npos - 1; s >= 0; --s) {
      const int r = w.rev ? npos - 1 - s : s;
      const float dl = to_f32(sDL[r * FB_DT + c]), dy = to_f32(sDY[r * FB_DT + c]);
      const float *row = sDB + r * Cp + n0, *rowC = sDC + r * Cp + n0;
      if (!MAIN) {
#pragma unroll
        for (int q = 0; q < NS / 4; ++q) {
          const float4 cv = *reinterpret_cast<const float4 *>(rowC + N + 4 * q);
          dh[4 * q] = fmaf(dy, cv.x, dh[4 * q]) * ex2(dl * a2[4 * q]);
          dh[4 * q + 1] = fmaf(dy, cv.y, dh[4 * q + 1]) * ex2(dl * a2[4 * q + 1]);
          dh[4 * q + 2] = fmaf(dy, cv.z, dh[4 * q + 2]) * ex2(dl * a2[4 * q + 2]);
          dh[4 * q + 3] = fmaf(dy, cv.w, dh[4 * q + 3]) * ex2(dl * a2[4 * q + 3]);
        }
        sumdl += dl;
        continue;
      }
      const float u = to_f32(sXC[r * FB_DT + c]);
      const float dlu = dl * u;
      float cB[NS], cC[NS];
      float s1 = 0.f, s2 = 0.f;     // Σ dh·B and Σ t·a2 over this lane's states
#pragma unroll
      for (int q = 0; q < NS / 4; ++q) {
        const float4 bv = *reinterpret_cast<const float4 *>(row + 4 * q);
        const float4 cv = *reinterpret_cast<const float4 *>(rowC + N + 4 * q);
        const float4 hv = sHt[(s * (NS / 4) + q) * NT];
        const float Bq[4] = {bv.x, bv.y, bv.z, bv.w}, Cq[4] = {cv.x, cv.y, cv.z, cv.w}, Hq[4] = {hv.x, hv.y, hv.z, hv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int sI = 4 * q + e;
          const float a = ex2(dl * a2[sI]);
          const float dhn = fmaf(dy, Cq[e], dh[sI]);          // gradient reaching h at this step
          cC[sI] = dy * Hq[e];                                 // dC term
          const float t = dhn * fmaf(-dlu, Bq[e], Hq[e]);      // dh · a·h_prev,  a·h_prev = h - delta·u·B
          s1 = fmaf(dhn, Bq[e], s1);
          s2 = fmaf(t, a2[sI], s2);
          dAt[sI] = fmaf(t, dl, dAt[sI]);
          cB[sI] = dhn * dlu;                                  // dB term
          dh[sI] = dhn * a;
        }
      }
      // dB / dC: sum over the CPW channels of this warp that share the lane's state set, one coalesced red per row
      int wb = 0, wc = 0;
      const float rB = transpose_reduce<NS, CPW / 2>(cB, lane, wb);
      const float rC = transpose_reduce<NS, CPW / 2>(cC, lane, wc);
      constexpr int DUP = CPW / NS;
      if ((cl & (DUP - 1)) == 0) {
        const long long pos = (long long)o * p.pso[w.k] + (long long)(i0 + r) * p.psi[w.k];
        if (DET) {
          const long long tile = (long long)blockIdx.x * (NT / 32) + warp;
          float *dst = p.part_bc + (((tile * p.batch + w.b) * p.Lseq + pos) * p.K + w.k) * 2 * N;
          dst[n0 + wb] = rB;
          dst[N + n0 + wb] = rC;
        } else {
          float *dst = dxrow0 + pos * p.K * Cp;
          float *dstC = CROSS ? dxrowC + pos * p.K * Cp : dst;
          atomicAdd(dst + n0 + wb, rB);
          atomicAdd(dstC + N + n0 + wb, rC);
        }
      }
      if (LPC == 2) {
        s1 += __shfl_xor_sync(0xffffffffu, s1, 16);
        s2 += __shfl_xor_sync(0xffffffffu, s2, 16);
      }
      float ddl = fmaf(u, s1, s2 * kLn2);
      const float duv = fmaf(dy, Dv, dl * s1);
      dDacc = fmaf(dy, u, dDacc);
      ddl *= 1.f - ex2(-dl * kLog2e);                          // softplus'(x) = sigmoid(x) = 1 - exp(-softplus(x))
      dbacc += ddl;
      if (half == 0) { sdu[r * CPW + cl] = duv; sdd[r * CPW + cl] = ddl; }
    }
    if (MAIN) {
#pragma unroll
      for (int s = 0; s < NS; ++s) dAacc[s] += dAt[s];
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) {
        if (DET) tma_store_4d(&p.m_dxc[w.k], sdu, w.d0 + warp * CPW, i0, o, w.k * p.batch + w.b);   // this direction's du slab
        else tma_reduce_add_4d(&p.m_dxc[w.k], sdu, w.d0 + warp * CPW, i0, o, w.b);
        tma_store_4d(&p.m_dd[w.k], sdd, w.d0 + warp * CPW, i0, o, w.k * p.batch + w.b);
        tma_store_commit();
        tma_store_wait_read<0>();
      }
    }
    __syncwarp();
    if (lane == 0 && kk + NST < ntl) {
      const uint32_t old = smem_inc_acq_rel(&done[st]);
      if ((old + 1) % (uint32_t)nwarps == 0) request_tile(kk + NST, st);
    }
    if (++st == NST) { st = 0; ph ^= 1; }
  }
  if (MAIN) {
    if (lane == 0) tma_store_wait_all<0>();
    if (DET) {
      const long long seg = (long long)w.b * p.nsplit + w.split;
#pragma unroll
      for (int s = 0; s < NS; ++s) p.part_dA[(seg * p.K * p.D + wd) * N + n0 + s] = dAacc[s];
      if (half == 0) { p.part_dD[seg * p.K * p.D + wd] = dDacc; p.part_db[seg * p.K * p.D + wd] = dbacc; }
    } else {
#pragma unroll
      for (int s = 0; s < NS; ++s) atomicAdd(&p.dA[wd * N + n0 + s], dAacc[s]);
      if (half == 0) {
        atomicAdd(&p.dDs[wd], dDacc);
        atomicAdd(&p.ddtb[wd], dbacc);
      }
    }
  } else {
#pragma unroll
    for (int s = 0; s < NS; ++s) { carry_row[n0 + s] = ex2(a2[s] * sumdl); carry_row[N + n0 + s] = dh[s]; }
  }
}

template <int N, int MODE>
__global__ void __launch_bounds__(128, 2) ss2d_bwd_kernel(const __grid_constant__ Ss2dBwdParams p) { ss2d_bwd_body<N, MODE, false, false>(p); }

template <int N, int MODE>
__global__ void __launch_bounds__(128, 2) ss2d_bwd_det_kernel(const __grid_constant__ Ss2dBwdParams p) { ss2d_bwd_body<N, MODE, true, false>(p); }

template <int N, int MODE>
__global__ void __launch_bounds__(128, 2) ss2d_bwd_cross_kernel(const __grid_constant__ Ss2dBwdParams p) { ss2d_bwd_body<N, MODE, false, true>(p); }

// the bf16 training mode (non-deterministic only): bf16 xc / dy / delta' tiles
template <int N, int MODE>
__global__ void __launch_bounds__(128, 2) ss2d_bwd_bf16_kernel(const __grid_constant__ Ss2dBwdParams p) { ss2d_bwd_body<N, MODE, false, false, __nv_bfloat16>(p); }

template <int N, int MODE>
__global__ void __launch_bounds__(128, 2) ss2d_bwd_cross_bf16_kernel(const __grid_constant__ Ss2dBwdParams p) { ss2d_bwd_body<N, MODE, false, true, __nv_bfloat16>(p); }

// the fp16 training mode (non-deterministic only): fp16 xc / dy / delta' tiles
template <int N, int MODE>
__global__ void __launch_bounds__(128, 2) ss2d_bwd_fp16_kernel(const __grid_constant__ Ss2dBwdParams p) { ss2d_bwd_body<N, MODE, false, false, __half>(p); }

template <int N, int MODE>
__global__ void __launch_bounds__(128, 2) ss2d_bwd_cross_fp16_kernel(const __grid_constant__ Ss2dBwdParams p) { ss2d_bwd_body<N, MODE, false, true, __half>(p); }

// ---- host ----
constexpr int kFbMaxSplit = 64;

// walks per image K (x_dbl rows per position) and parameter sets (K, or the 2 modalities of CROSS)
static int fb_dirs(int kind) { return kind == SIGMA_DIRS_CROSS4 ? 4 : (kind == SIGMA_DIRS_SEQ2 ? 2 : 1); }
static int fb_wsets(int kind) { return kind == SIGMA_DIRS_CROSS ? 2 : fb_dirs(kind); }

static int fb_max_tiles(int kind, int H, int W) { return ss2d_save_tiles(kind, H, W); }
int ss2d_save_tiles(int kind, int H, int W) {
  const long long L = (long long)H * W;
  if (kind == SIGMA_DIRS_SEQ2) return (int)((2 * L + FB_LT - 1) / FB_LT);
  if (kind == SIGMA_DIRS_CROSS) return (int)((L + FB_LT - 1) / FB_LT);   // one row-major walk
  return (int)std::max<long long>((L + FB_LT - 1) / FB_LT, (long long)W * ((H + FB_LT - 1) / FB_LT));
}

size_t ss2d_scan_hs_bytes(int kind, int batch, int H, int W, int D, int N) {
  const int K = fb_dirs(kind);
  return (size_t)K * batch * fb_max_tiles(kind, H, W) * D * N * sizeof(float);
}

// workspace = [reverse carries (batch, K, D, 64 segments, 2N)]
size_t ss2d_scan_bwd_workspace_bytes(int kind, int batch, int H, int W, int D, int N) {
  return align256((size_t)batch * fb_dirs(kind) * D * kFbMaxSplit * 2 * N * sizeof(float));
}

// the deterministic build appends [du slabs (K, batch, Lseq, D)] [dB / dC partials (D / CPW, batch, Lseq, K, 2N)]
// [dA partials (batch·64, K·D, N)] [dDs partials (batch·64, K·D)] [d dt_bias partials (batch·64, K·D)]
struct FbDetLayout { size_t du, bc, dA, dD, total; };

static FbDetLayout fb_det_layout(int kind, int batch, int H, int W, int D, int N) {
  const int K = kind == SIGMA_DIRS_CROSS4 ? 4 : 2, CPW = N >= 16 ? 16 : 32;
  const size_t Lseq = kind == SIGMA_DIRS_SEQ2 ? 2ull * H * W : (size_t)H * W;
  const size_t segs = (size_t)batch * kFbMaxSplit;
  FbDetLayout l;
  l.du = ss2d_scan_bwd_workspace_bytes(kind, batch, H, W, D, N);
  l.bc = l.du + align256((size_t)K * batch * Lseq * D * sizeof(float));
  l.dA = l.bc + align256((size_t)(D / CPW) * batch * Lseq * K * 2 * N * sizeof(float));
  l.dD = l.dA + align256(segs * K * D * N * sizeof(float));
  l.total = l.dD + 2 * align256(segs * K * D * sizeof(float));
  return l;
}

size_t ss2d_scan_bwd_det_workspace_bytes(int kind, int batch, int H, int W, int D, int N) {
  return fb_det_layout(kind, batch, H, W, D, N).total;
}

// The L-segment plan of both sweeps.  All directions share tiles_per_split, so a direction with fewer tiles than the
// longest walk (min_tiles < max_tiles) can get empty trailing segments.  force_split > 0 overrides the count (capped at 64).
struct FbPlan { int nsplit, tiles_per_split, max_tiles, min_tiles; };

static FbPlan fb_plan(int kind, int batch, int H, int W, int D, int N, int force_split) {
  const int K = fb_dirs(kind);
  const long long Lseq = kind == SIGMA_DIRS_SEQ2 ? 2LL * H * W : (long long)H * W;
  const int row_tiles = (int)((Lseq + FB_LT - 1) / FB_LT), col_tiles = W * ((H + FB_LT - 1) / FB_LT);
  FbPlan pl;
  pl.max_tiles = kind == SIGMA_DIRS_CROSS4 ? std::max(row_tiles, col_tiles) : row_tiles;
  pl.min_tiles = kind == SIGMA_DIRS_CROSS4 ? std::min(row_tiles, col_tiles) : row_tiles;
  const int lpc = N >= 16 ? 2 : 1;
  int nsplit = pick_segments((long long)(D / FB_DT) * K * batch, pl.max_tiles, kNumSMs * (lpc == 2 ? 2 : 4), 1.3, kFbMaxSplit);
  if (force_split > 0) nsplit = std::min(force_split, kFbMaxSplit);
  nsplit = std::max(1, std::min(nsplit, pl.max_tiles));
  pl.tiles_per_split = (pl.max_tiles + nsplit - 1) / nsplit;
  pl.nsplit = (pl.max_tiles + pl.tiles_per_split - 1) / pl.tiles_per_split;
  return pl;
}

int ss2d_bwd_plan_hook(int kind, int batch, int H, int W, int D, int N, int force_split, long long *out4) {
  const FbPlan pl = fb_plan(kind, batch, H, W, D, N, force_split);
  out4[0] = pl.nsplit; out4[1] = pl.tiles_per_split; out4[2] = pl.max_tiles; out4[3] = pl.min_tiles;
  return SIGMA_OK;
}

// delta / ddelta: (K, batch, Lseq, D) slabs stored at the position a value belongs to; dxc (batch, Lseq, D) and dxdbl
// (batch, Lseq, K, Cp) are ACCUMULATED INTO after being zeroed here; dA (K·D, N), dDs (K·D), ddtb (K, D) overwritten.
// det: the main sweep writes partials (see fb_det_layout) that sum_parts_det_kernel adds in a fixed order.
// xdtype: element type of xc, dy and delta (SIGMA_F32, or SIGMA_BF16 / SIGMA_F16 behind the float pointers; never with det, the
// entry points check)
int ss2d_scan_bwd(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A, const float *Ds,
                  const float *dy, const float *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl, float *dA, float *dDs,
                  float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *ws, size_t ws_bytes, int force_split,
                  cudaStream_t stream, int det, int xdtype) {
  const size_t need = det ? ss2d_scan_bwd_det_workspace_bytes(kind, batch, H, W, D, N) : ss2d_scan_bwd_workspace_bytes(kind, batch, H, W, D, N);
  if (ws == nullptr || ws_bytes < need) {
    set_error("sigma_ss2d_scan_bwd_saved: workspace too small (%zu < %zu)", ws_bytes, need);
    return SIGMA_EWORKSPACE;
  }
  const bool cross = kind == SIGMA_DIRS_CROSS;   // never with det (the entry points reject it)
  const uint64_t xes = xdtype == SIGMA_F32 ? 4 : 2;   // bytes per xc / dy / delta element
  Ss2dBwdParams p;
  memset(&p, 0, sizeof(p));
  const int K = fb_dirs(kind), Kw = fb_wsets(kind);
  const long long Lseq = kind == SIGMA_DIRS_SEQ2 ? 2LL * H * W : (long long)H * W;
  p.dtw = dtw; p.dtb = dtb; p.A = A; p.Ds = Ds; p.hs = hs;
  p.dxdbl = dxdbl; p.dA = dA; p.dDs = dDs; p.ddtb = ddtb;
  p.D = D; p.N = N; p.R = R; p.Cp = Cp; p.K = K; p.batch = batch; p.Lseq = Lseq;
  p.max_tiles = fb_max_tiles(kind, H, W);
  p.carry = (float *)ws;
  // The zeroing comes before the tensor maps: it is the call's first runtime API call, which binds the device's primary context
  // to a thread that has none yet (autograd runs a backward that starts at this node on its own thread), and
  // cuTensorMapEncodeTiled fails without a current context.
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dxc, 0, (size_t)batch * Lseq * D * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dxdbl, 0, (size_t)batch * Lseq * K * Cp * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dA, 0, (size_t)Kw * D * N * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dDs, 0, (size_t)Kw * D * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(ddtb, 0, (size_t)Kw * D * sizeof(float), stream));
  const int CPW = N >= 16 ? 16 : 32;
  int rc;
  auto tmap = [](CUtensorMap *map, const void *base, const uint64_t *dims, const uint64_t *str, const uint32_t *box,
                 CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT32) {
    return make_tmap(map, dtype, 4, base, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  };
  const CUtensorMapDataType xdt = xdtype == SIGMA_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                  : xdtype == SIGMA_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  for (int k = 0; k < K; ++k) {
    const bool colmajor = kind == SIGMA_DIRS_CROSS4 && (k & 1);
    p.rev[k] = kind == SIGMA_DIRS_CROSS4 ? (k >= 2) : (k == 1);
    uint64_t dims[4], str[3], strx[3];   // str: fp32 rows (dxc); strx: rows of xc / dy / delta
    uint32_t box[4] = {(uint32_t)FB_DT, (uint32_t)FB_LT, 1, 1}, boxw[4] = {(uint32_t)CPW, (uint32_t)FB_LT, 1, 1};
    if (!colmajor) {
      p.I[k] = (int)Lseq; p.O[k] = 1; p.psi[k] = 1; p.pso[k] = 0;
      dims[0] = D; dims[1] = Lseq; dims[2] = 1; dims[3] = batch;
      str[0] = (uint64_t)D * 4; str[1] = (uint64_t)Lseq * D * 4; str[2] = (uint64_t)Lseq * D * 4;
    } else {   // inner index h at fixed w: position h·W + w
      p.I[k] = H; p.O[k] = W; p.psi[k] = W; p.pso[k] = 1;
      dims[0] = D; dims[1] = H; dims[2] = W; dims[3] = batch;
      str[0] = (uint64_t)W * D * 4; str[1] = (uint64_t)D * 4; str[2] = (uint64_t)Lseq * D * 4;
    }
    for (int i = 0; i < 3; ++i) strx[i] = str[i] / 4 * xes;
    if ((rc = tmap(&p.m_xc[k], xc, dims, strx, box, xdt))) return rc;
    if ((rc = tmap(&p.m_dy[k], dy, dims, strx, box, xdt))) return rc;
    if ((rc = tmap(&p.m_dxc[k], dxc, dims, str, boxw))) return rc;
    dims[3] = (uint64_t)K * batch;   // slabs: image index k·batch + b
    if ((rc = tmap(&p.m_dl[k], delta, dims, strx, box, xdt))) return rc;
    dims[3] = batch;
    uint32_t boxd[4] = {(uint32_t)Cp, (uint32_t)FB_LT, 1, 1};
    dims[0] = Cp;
    const uint64_t pos = (uint64_t)K * Cp * 4;
    if (!colmajor) { str[0] = pos; str[1] = Lseq * pos; str[2] = Lseq * pos; }
    else { str[0] = W * pos; str[1] = pos; str[2] = Lseq * pos; }
    if ((rc = tmap(&p.m_dbl[k], xdbl + (long long)k * Cp, dims, str, boxd))) return rc;
  }
  const FbPlan pl = fb_plan(kind, batch, H, W, D, N, force_split);
  p.tiles_per_split = pl.tiles_per_split;
  p.nsplit = pl.nsplit;
  p.nst = 2;

  // per-warp boxes over (K, batch, Lseq, D) slabs: m_dd over ddelta, and for det m_dxc over the du slabs
  auto make_dd = [&](float *slab, CUtensorMap *maps = nullptr) -> int {
    for (int k = 0; k < K; ++k) {
      const bool colmajor = kind == SIGMA_DIRS_CROSS4 && (k & 1);
      uint64_t dims[4], str[3];
      uint32_t boxw[4] = {(uint32_t)CPW, (uint32_t)FB_LT, 1, 1};
      if (!colmajor) {
        dims[0] = D; dims[1] = Lseq; dims[2] = 1; dims[3] = (uint64_t)K * batch;
        str[0] = (uint64_t)D * 4; str[1] = (uint64_t)Lseq * D * 4; str[2] = (uint64_t)Lseq * D * 4;
      } else {
        dims[0] = D; dims[1] = H; dims[2] = W; dims[3] = (uint64_t)K * batch;
        str[0] = (uint64_t)W * D * 4; str[1] = (uint64_t)D * 4; str[2] = (uint64_t)Lseq * D * 4;
      }
      int r = tmap(maps ? &maps[k] : &p.m_dd[k], slab, dims, str, boxw);
      if (r) return r;
    }
    return SIGMA_OK;
  };
  if ((rc = make_dd(ddelta))) return rc;
  const FbDetLayout dl = fb_det_layout(kind, batch, H, W, D, N);
  float *du_slabs = (float *)((char *)ws + dl.du);
  if (det) {   // du goes to per-direction slabs (plain TMA stores with the slab maps), the partials to the workspace
    if ((rc = make_dd(du_slabs, p.m_dxc))) return rc;
    p.part_bc = (float *)((char *)ws + dl.bc);
    p.part_dA = (float *)((char *)ws + dl.dA);
    p.part_dD = (float *)((char *)ws + dl.dD);
    p.part_db = p.part_dD + (size_t)batch * kFbMaxSplit * K * D;
  }
  auto go = [&](auto tag) -> int {
    constexpr int NN = decltype(tag)::value;
    constexpr int LPC = FbCfg<NN>::LPC, NS = FbCfg<NN>::NS, CPWc = FbCfg<NN>::CPW, NT = FB_DT * LPC;
    dim3 grid(D / FB_DT, K * p.nsplit, batch), block(NT);
    const long long nrows = (long long)batch * K * D, tot = nrows * NN;
    const size_t dbl_tiles = cross ? 2 : 1;   // the reverse sweeps of CROSS also stage the C image's x_dbl tile
    const size_t xt_fl = FB_LT * FB_DT * xes / 4;   // an xc / dy / delta tile, in floats
    const size_t sm_smem = ((size_t)p.nst * (2 * xt_fl + dbl_tiles * FB_LT * Cp)) * sizeof(float) + 256;
    const size_t mn_smem = ((size_t)p.nst * (3 * xt_fl + dbl_tiles * FB_LT * Cp) + (NT / 32) * 2 * FB_LT * CPWc + (size_t)FB_LT * NS * NT) * sizeof(float) + 256;
    auto run = [&](auto kern, size_t smem) -> int {
      SIGMA_CHECK_CUDA(prep_kernel_once((const void *)kern));
      kern<<<grid, block, smem, stream>>>(p);
      SIGMA_CHECK_LAUNCH();
      return SIGMA_OK;
    };
    using Kern = void (*)(Ss2dBwdParams);
    auto pick = [&](auto mode) -> Kern {
      constexpr int M = decltype(mode)::value;
      if (xdtype == SIGMA_BF16) return cross ? ss2d_bwd_cross_bf16_kernel<NN, M> : ss2d_bwd_bf16_kernel<NN, M>;
      if (xdtype == SIGMA_F16) return cross ? ss2d_bwd_cross_fp16_kernel<NN, M> : ss2d_bwd_fp16_kernel<NN, M>;
      return cross ? ss2d_bwd_cross_kernel<NN, M> : ss2d_bwd_kernel<NN, M>;
    };
    const Kern bw_serial = pick(std::integral_constant<int, MODE_SERIAL>{});
    const Kern bw_summary = pick(std::integral_constant<int, MODE_SUMMARY>{});
    const Kern bw_apply = pick(std::integral_constant<int, MODE_APPLY>{});
    int r;
    if (!det) {
      if (p.nsplit == 1) return run(bw_serial, mn_smem);
      if ((r = run(bw_summary, sm_smem))) return r;
      scan_combine_rev_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(p.carry, nrows, p.nsplit, NN);
      SIGMA_CHECK_LAUNCH();
      return run(bw_apply, mn_smem);
    }
    if (p.nsplit == 1) {
      if ((r = run(ss2d_bwd_det_kernel<NN, MODE_SERIAL>, mn_smem))) return r;
    } else {
      if ((r = run(ss2d_bwd_kernel<NN, MODE_SUMMARY>, sm_smem))) return r;
      scan_combine_rev_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(p.carry, nrows, p.nsplit, NN);
      SIGMA_CHECK_LAUNCH();
      if ((r = run(ss2d_bwd_det_kernel<NN, MODE_APPLY>, mn_smem))) return r;
    }
    // fixed-order sums: du over directions k, dB / dC over warp channel tiles, dA / dDs / d dt_bias over (image, segment)
    const int segs = batch * p.nsplit;
    const long long KD = (long long)K * D;
    if ((r = sum_parts_det_launch(du_slabs, K, (long long)batch * Lseq * D, (long long)batch * Lseq * D, 0, dxc, stream))) return r;
    if ((r = sum_parts_det_launch(p.part_bc, D / CPWc, (long long)batch * Lseq * K * 2 * NN, 2 * NN, Cp, dxdbl, stream))) return r;
    if ((r = sum_parts_det_launch(p.part_dA, segs, KD * NN, KD * NN, 0, dA, stream))) return r;
    if ((r = sum_parts_det_launch(p.part_dD, segs, KD, KD, 0, dDs, stream))) return r;
    return sum_parts_det_launch(p.part_db, segs, KD, KD, 0, ddtb, stream);
  };
  if (N == 16) return go(std::integral_constant<int, 16>{});
  return go(std::integral_constant<int, 4>{});
}

}  // namespace sigma
