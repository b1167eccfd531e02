// a3 — op-level selective scan backward, GENERIC path (shapes TMA cannot express: ragged rows, channel groups that are
// not a multiple of 32; d_state <= 16).  Every Sigma call takes scan_op_bwd_tma.cu instead.
// (reference: csrc/selective_scan/selective_scan.cpp:251-362, selective_scan_bwd_kernel.cuh:68-274).
// fp16 / bf16 inputs and du / ddelta outputs are read / written natively.
//
// Two sweeps.  (1) The forward kernel re-runs with `hs` set and leaves the state at the start of every
// 32-position tile in scratch (the reference recomputes from its 2048-chunk states `x`, bwd_kernel.cuh:114-116).
// (2) This kernel walks the tiles BACKWARDS: per tile it recomputes h inside the tile from the checkpoint
// (kept in shared memory, one row per position), then runs the reverse recurrence
//     dh_l = a_{l+1}·dh_{l+1} + dout_l·C_l
// producing du, ddelta (softplus' applied), and the per-thread dA; dB/dC are reduced over the CTA's 32 channels
// with warp shuffles + shared-memory adds and leave the CTA as ONE atomicAdd per (n, l) — the reference issues one
// per channel (bwd_kernel.cuh:214-227: 192..1536-way contention on the same address).
// Thread mapping as the forward: LPC lanes per channel, SPT = 4 states per lane.
#include <algorithm>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "scan_core.cuh"

namespace sigma {

constexpr int BW_LT = 32, BW_LTP = 36, BW_DT = 32;

struct ScanBwdParams {
  const void *u, *delta, *B, *C, *dout;   // element type T
  const float *A, *D, *bias, *hs;
  void *du, *ddelta;                      // element type T
  float *dA, *dB, *dC, *dD, *dbias;
  int batch, dim, L, N, G, dpg, tiles_per_group, ntiles, softplus;
  // deterministic build (scan_op_bwd_det_kernel): dB / dC partials per CTA channel tile of a group (tiles_per_group, batch,
  // G, N, L); dA (batch, dim, N), dD and ddelta_bias (batch, dim) per batch
  float *part_B, *part_C, *part_dA, *part_dD, *part_db;
};

template <int SPT, int LPC>
__host__ __device__ constexpr int bwd_smem_floats() {
  // inputs: u, delta, dout (32 rows each) + B, C (NP rows each); outputs: du, ddelta (32 rows), dB, dC (NP rows);
  // h rows: 32 positions x (32*LPC threads) x SPT
  return (3 * BW_DT + 2 * SPT * LPC) * BW_LTP + (2 * BW_DT + 2 * SPT * LPC) * BW_LTP + BW_LT * 32 * LPC * SPT;
}

// DET: the warps' dB / dC rows go to per-warp shared-memory slots summed in warp order (after the h rows), the CTA's sums
// and the per-thread dA / dD / ddelta_bias to the partials of the deterministic build (see ScanBwdParams)
template <typename T, int SPT, int LPC, bool DET>
__device__ __forceinline__ void scan_op_bwd_body(const ScanBwdParams &p) {
  const T *pu = (const T *)p.u, *pdl = (const T *)p.delta, *pdo = (const T *)p.dout, *pB = (const T *)p.B, *pC = (const T *)p.C;
  constexpr int NP = SPT * LPC, CPW = 32 / LPC, NTH = 32 * LPC;
  extern __shared__ __align__(16) float smem[];
  float *sU = smem, *sDl = sU + BW_DT * BW_LTP, *sDo = sDl + BW_DT * BW_LTP;
  float *sB = sDo + BW_DT * BW_LTP, *sC = sB + NP * BW_LTP;
  float *sDu = sC + NP * BW_LTP, *sDd = sDu + BW_DT * BW_LTP;
  float *sDB = sDd + BW_DT * BW_LTP, *sDC = sDB + NP * BW_LTP;
  float *sH = sDC + NP * BW_LTP;  // [position][thread][SPT]
  float *sBCw = sH + BW_LT * NTH * SPT;   // DET: [warp][dB rows | dC rows]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q = lane % LPC, c_local = warp * CPW + lane / LPC;
  const int g = blockIdx.x / p.tiles_per_group, tg = blockIdx.x - g * p.tiles_per_group;
  const int d_in_g0 = tg * BW_DT, d0 = g * p.dpg + d_in_g0;
  const int nch = min(BW_DT, p.dpg - d_in_g0);
  const bool ch_ok = c_local < nch;
  const int d = d0 + (ch_ok ? c_local : 0);
  const int b = blockIdx.y;
  const long long row0 = ((long long)b * p.dim + d0) * p.L;          // contiguous (batch, dim, L)
  const long long bc0 = ((long long)b * p.G + g) * p.N * (long long)p.L;

  float a2[SPT], Araw[SPT], dh[SPT], dAacc[SPT];
#pragma unroll
  for (int s = 0; s < SPT; ++s) {
    const int n = q * SPT + s;
    Araw[s] = (ch_ok && n < p.N) ? p.A[(long long)d * p.N + n] : 0.f;
    a2[s] = Araw[s] * kLog2e;
    dh[s] = 0.f;
    dAacc[s] = 0.f;
  }
  const float bias = (p.bias && ch_ok) ? p.bias[d] : 0.f;
  const float Dv = (p.D && ch_ok) ? p.D[d] : 0.f;
  float dDacc = 0.f, dbacc = 0.f;

  for (int t = p.ntiles - 1; t >= 0; --t) {
    const int l0 = t * BW_LT, npos = min(BW_LT, p.L - l0);
    // ---- load the tile (plain loads; the backward is not the headline path) ----
    for (int i = tid; i < (3 * BW_DT + 2 * NP) * BW_LT; i += NTH) {
      const int row = i >> 5, e = i & 31;
      float v = 0.f;
      if (e < npos) {
        if (row < BW_DT) { if (row < nch) v = to_f32(pu[row0 + (long long)row * p.L + l0 + e]); }
        else if (row < 2 * BW_DT) { if (row - BW_DT < nch) v = to_f32(pdl[row0 + (long long)(row - BW_DT) * p.L + l0 + e]); }
        else if (row < 3 * BW_DT) { if (row - 2 * BW_DT < nch) v = to_f32(pdo[row0 + (long long)(row - 2 * BW_DT) * p.L + l0 + e]); }
        else if (row < 3 * BW_DT + NP) { const int n = row - 3 * BW_DT; if (n < p.N) v = to_f32(pB[bc0 + (long long)n * p.L + l0 + e]); }
        else { const int n = row - 3 * BW_DT - NP; if (n < p.N) v = to_f32(pC[bc0 + (long long)n * p.L + l0 + e]); }
      }
      smem[row * BW_LTP + e] = v;
    }
    for (int i = tid; i < 2 * NP * BW_LTP; i += NTH) sDB[i] = 0.f;   // sDB and sDC are adjacent
    __syncthreads();

    // ---- forward recompute inside the tile, keeping h after every position ----
    float h[SPT];
    const float *hs_row = p.hs + (((long long)b * p.dim + d) * p.ntiles + t) * NP + q * SPT;
#pragma unroll
    for (int s = 0; s < SPT; ++s) h[s] = ch_ok ? hs_row[s] : 0.f;
    float hstart[SPT];
#pragma unroll
    for (int s = 0; s < SPT; ++s) hstart[s] = h[s];
    for (int i = 0; i < npos; ++i) {
      const float raw = sDl[c_local * BW_LTP + i] + bias;
      const float dl = p.softplus ? softplus20(raw) : raw;
      const float dlu = dl * sU[c_local * BW_LTP + i];
#pragma unroll
      for (int s = 0; s < SPT; ++s) {
        h[s] = fmaf(ex2(dl * a2[s]), h[s], dlu * sB[(q * SPT + s) * BW_LTP + i]);
        sH[((long long)i * NTH + tid) * SPT + s] = h[s];
      }
    }

    // ---- reverse recurrence (dA: per-tile partial sums folded into the running total — two-level summation) ----
    float dAt[SPT];
#pragma unroll
    for (int s = 0; s < SPT; ++s) dAt[s] = 0.f;
    for (int i = npos - 1; i >= 0; --i) {
      const float raw = sDl[c_local * BW_LTP + i] + bias;
      const float dl = p.softplus ? softplus20(raw) : raw;
      const float ui = sU[c_local * BW_LTP + i];
      const float dy = sDo[c_local * BW_LTP + i];
      float ddl = 0.f, dui = 0.f;
      float cB[SPT], cC[SPT];
#pragma unroll
      for (int s = 0; s < SPT; ++s) {
        const float Bn = sB[(q * SPT + s) * BW_LTP + i], Cn = sC[(q * SPT + s) * BW_LTP + i];
        const float hi = sH[((long long)i * NTH + tid) * SPT + s];
        const float hprev = i > 0 ? sH[((long long)(i - 1) * NTH + tid) * SPT + s] : hstart[s];
        const float a = ex2(dl * a2[s]);
        dh[s] = fmaf(dy, Cn, dh[s]);                 // gradient reaching h_i (bwd_kernel.cuh:173-199)
        cC[s] = dy * hi;                              // dC contribution (:225)
        const float da = dh[s] * hprev;               // d/da of a·h_{i-1}
        ddl = fmaf(da * a, Araw[s], fmaf(dh[s] * Bn, ui, ddl));   // (:206)
        dAt[s] = fmaf(da * a, dl, dAt[s]);            // (:208)
        cB[s] = dh[s] * dl * ui;                      // dB contribution (:224)
        dui = fmaf(dh[s] * dl, Bn, dui);              // (:205)
        dh[s] *= a;
      }
      // dB / dC: sum over the channels of this warp (lanes that share q), then one shared-memory add per warp
#pragma unroll
      for (int s = 0; s < SPT; ++s) {
#pragma unroll
        for (int o = LPC; o < 32; o <<= 1) {
          cB[s] += __shfl_xor_sync(0xffffffffu, cB[s], o);
          cC[s] += __shfl_xor_sync(0xffffffffu, cC[s], o);
        }
      }
      if (lane < LPC) {
#pragma unroll
        for (int s = 0; s < SPT; ++s) {
          if (DET) {
            sBCw[(warp * 2 * NP + q * SPT + s) * BW_LTP + i] = cB[s];
            sBCw[(warp * 2 * NP + NP + q * SPT + s) * BW_LTP + i] = cC[s];
          } else {
            atomicAdd(&sDB[(q * SPT + s) * BW_LTP + i], cB[s]);
            atomicAdd(&sDC[(q * SPT + s) * BW_LTP + i], cC[s]);
          }
        }
      }
      ddl = channel_reduce<LPC>(ddl);
      dui = channel_reduce<LPC>(dui);
      if (q == 0) {
        dui = fmaf(dy, Dv, dui);                                        // (:143,250)
        dDacc = fmaf(dy, ui, dDacc);                                    // (:144)
        if (p.softplus && raw <= 20.f) ddl *= __fdividef(1.f, 1.f + ex2(-raw * kLog2e));   // (:241-245)
        dbacc += ddl;
        sDu[c_local * BW_LTP + i] = dui;
        sDd[c_local * BW_LTP + i] = ddl;
      }
    }
#pragma unroll
    for (int s = 0; s < SPT; ++s) dAacc[s] += dAt[s];
    __syncthreads();
    // ---- write the tile: du, ddelta rows; dB/dC: one atomic per (n, l) per CTA ----
    for (int i = tid; i < 2 * BW_DT * BW_LT; i += NTH) {
      const int which = i / (BW_DT * BW_LT), r = (i >> 5) % BW_DT, e = i & 31;
      if (r < nch && e < npos) {
        T *dst = (T *)(which ? p.ddelta : p.du);
        dst[row0 + (long long)r * p.L + l0 + e] = from_f32<T>((which ? sDd : sDu)[r * BW_LTP + e]);
      }
    }
    for (int i = tid; i < 2 * NP * BW_LT; i += NTH) {
      const int which = i / (NP * BW_LT), n = (i >> 5) % NP, e = i & 31;
      if (n < p.N && e < npos) {
        if (DET) {
          float v = 0.f;
#pragma unroll
          for (int wp = 0; wp < NTH / 32; ++wp) v += sBCw[(wp * 2 * NP + which * NP + n) * BW_LTP + e];
          const long long po = (long long)tg * p.batch * p.G * p.N * p.L + bc0 + (long long)n * p.L + l0 + e;
          (which ? p.part_C : p.part_B)[po] = v;
        } else {
          atomicAdd((which ? p.dC : p.dB) + bc0 + (long long)n * p.L + l0 + e, (which ? sDC : sDB)[n * BW_LTP + e]);
        }
      }
    }
    __syncthreads();
  }
  if (DET && ch_ok) {
    const long long bd = (long long)b * p.dim + d;
#pragma unroll
    for (int s = 0; s < SPT; ++s) {
      const int n = q * SPT + s;
      if (n < p.N) p.part_dA[bd * p.N + n] = dAacc[s];
    }
    if (q == 0) {
      if (p.dD) p.part_dD[bd] = dDacc;
      if (p.dbias) p.part_db[bd] = dbacc;
    }
  } else if (ch_ok) {
#pragma unroll
    for (int s = 0; s < SPT; ++s) {
      const int n = q * SPT + s;
      if (n < p.N) atomicAdd(&p.dA[(long long)d * p.N + n], dAacc[s]);   // over batch (:262-273)
    }
    if (q == 0) {
      if (p.dD) atomicAdd(&p.dD[d], dDacc);
      if (p.dbias) atomicAdd(&p.dbias[d], dbacc);
    }
  }
}

template <typename T, int SPT, int LPC>
__global__ void __launch_bounds__(32 * LPC) scan_op_bwd_kernel(const ScanBwdParams p) { scan_op_bwd_body<T, SPT, LPC, false>(p); }

template <typename T, int SPT, int LPC>
__global__ void __launch_bounds__(32 * LPC) scan_op_bwd_det_kernel(const ScanBwdParams p) { scan_op_bwd_body<T, SPT, LPC, true>(p); }

template <typename T, int SPT, int LPC>
static int launch_bwd(const ScanBwdParams &p, cudaStream_t stream) {
  const bool det = p.part_B != nullptr;
  const size_t smem = (size_t)(bwd_smem_floats<SPT, LPC>() + (det ? LPC * 2 * SPT * LPC * BW_LTP : 0)) * sizeof(float);
  auto kern = det ? scan_op_bwd_det_kernel<T, SPT, LPC> : scan_op_bwd_kernel<T, SPT, LPC>;
  SIGMA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(p.G * p.tiles_per_group, p.batch);
  kern<<<grid, 32 * LPC, smem, stream>>>(p);
  SIGMA_CHECK_LAUNCH();
  if (!det) return SIGMA_OK;
  // fixed-order sums: dB / dC over the channel tiles of a group, dA / dD / ddelta_bias over the batch
  const long long bgnl = (long long)p.batch * p.G * p.N * p.L, dn = (long long)p.dim * p.N;
  int rc;
  if ((rc = sum_parts_det_launch(p.part_B, p.tiles_per_group, bgnl, bgnl, 0, p.dB, stream))) return rc;
  if ((rc = sum_parts_det_launch(p.part_C, p.tiles_per_group, bgnl, bgnl, 0, p.dC, stream))) return rc;
  if ((rc = sum_parts_det_launch(p.part_dA, p.batch, dn, dn, 0, p.dA, stream))) return rc;
  if (p.dD && (rc = sum_parts_det_launch(p.part_dD, p.batch, p.dim, p.dim, 0, p.dD, stream))) return rc;
  if (p.dbias && (rc = sum_parts_det_launch(p.part_db, p.batch, p.dim, p.dim, 0, p.dbias, stream))) return rc;
  return SIGMA_OK;
}

// scratch of the deterministic build: [dB partials] [dC partials] (tiles_per_group, batch, G, N, L) [dA partials (batch, dim, N)]
// [dD partials] [ddelta_bias partials] (batch, dim)
size_t scan_op_bwd_det_bytes(int batch, int dim, int L, int N, int G) {
  const size_t tpg = (size_t)(dim / G + BW_DT - 1) / BW_DT;
  return 2 * align256(tpg * batch * G * N * L * sizeof(float)) + align256((size_t)batch * dim * N * sizeof(float)) +
         2 * align256((size_t)batch * dim * sizeof(float));
}

size_t scan_op_bwd_workspace_bytes(int batch, int dim, int L, int N, int elem_bytes) {
  const size_t ntiles = (L + BW_LT - 1) / BW_LT;
  const size_t hs = (size_t)batch * dim * ntiles * scan_op_npad(N) * sizeof(float);
  const size_t out = (size_t)batch * dim * L * elem_bytes;   // forward output of the recompute sweep (discarded)
  return align256(hs) + align256(out);
}

// all tensors contiguous, element type T
template <typename T>
int scan_op_bwd_generic(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                        const float *bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                        float *dD, float *dbias, int batch, int dim, int L, int N, int G, int softplus, void *ws,
                        size_t ws_bytes, cudaStream_t stream, void *det_ws) {
  if (N > 16) { set_error("sigma_scan_bwd: d_state=%d > 16 is not supported by the backward kernels", N); return SIGMA_EUNSUPPORTED; }
  if (ws == nullptr || ws_bytes < scan_op_bwd_workspace_bytes(batch, dim, L, N, (int)sizeof(T))) {
    set_error("sigma_scan_bwd: workspace too small (%zu < %zu)", ws_bytes, scan_op_bwd_workspace_bytes(batch, dim, L, N, (int)sizeof(T)));
    return SIGMA_EWORKSPACE;
  }
  const int NP = scan_op_npad(N);
  const int ntiles = (L + BW_LT - 1) / BW_LT;
  float *hs = (float *)ws;
  const size_t hs_b = align256((size_t)batch * dim * ntiles * NP * sizeof(float));
  void *out_tmp = (char *)ws + hs_b;
  sigma_scan_strides st;
  st.u_batch = st.delta_batch = st.out_batch = (int64_t)dim * L;
  st.u_dim = st.delta_dim = st.out_dim = L;
  st.A_dim = N; st.A_dstate = 1;
  st.B_batch = st.C_batch = (int64_t)G * N * L;
  st.B_group = st.C_group = (int64_t)N * L;
  st.B_dstate = st.C_dstate = L;
  int rc = scan_op_fwd_generic<T>(u, delta, A, B, C, D, bias, out_tmp, nullptr, hs, batch, dim, L, N, G, softplus, st, nullptr, 0,
                                  1, stream);
  if (rc) return rc;
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dA, 0, (size_t)dim * N * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dB, 0, (size_t)batch * G * N * L * sizeof(float), stream));
  SIGMA_CHECK_CUDA(cudaMemsetAsync(dC, 0, (size_t)batch * G * N * L * sizeof(float), stream));
  if (dD) SIGMA_CHECK_CUDA(cudaMemsetAsync(dD, 0, (size_t)dim * sizeof(float), stream));
  if (dbias) SIGMA_CHECK_CUDA(cudaMemsetAsync(dbias, 0, (size_t)dim * sizeof(float), stream));
  ScanBwdParams p;
  p.u = u; p.delta = delta; p.A = A; p.B = B; p.C = C; p.D = D; p.bias = bias; p.dout = dout; p.hs = hs;
  p.du = du; p.ddelta = ddelta; p.dA = dA; p.dB = dB; p.dC = dC; p.dD = dD; p.dbias = dbias;
  p.batch = batch; p.dim = dim; p.L = L; p.N = N; p.G = G; p.dpg = dim / G;
  p.tiles_per_group = (p.dpg + BW_DT - 1) / BW_DT;
  p.ntiles = ntiles; p.softplus = softplus;
  p.part_B = p.part_C = p.part_dA = p.part_dD = p.part_db = nullptr;
  if (det_ws) {   // layout of scan_op_bwd_det_bytes
    const size_t bc = align256((size_t)p.tiles_per_group * batch * G * N * L * sizeof(float));
    const size_t da = align256((size_t)batch * dim * N * sizeof(float)), dd = align256((size_t)batch * dim * sizeof(float));
    char *w = (char *)det_ws;
    p.part_B = (float *)w; p.part_C = (float *)(w + bc); p.part_dA = (float *)(w + 2 * bc);
    p.part_dD = (float *)(w + 2 * bc + da); p.part_db = (float *)(w + 2 * bc + da + dd);
  }
  switch (NP) {
    case 4: return launch_bwd<T, 4, 1>(p, stream);
    case 8: return launch_bwd<T, 4, 2>(p, stream);
    default: return launch_bwd<T, 4, 4>(p, stream);
  }
}

#define SIGMA_INST(T)                                                                                                       \
  template int scan_op_bwd_generic<T>(const void *, const void *, const float *, const void *, const void *, const float *, \
                                      const float *, const void *, void *, void *, float *, float *, float *, float *,     \
                                      float *, int, int, int, int, int, int, void *, size_t, cudaStream_t, void *);
SIGMA_INST(float)
SIGMA_INST(__half)
SIGMA_INST(__nv_bfloat16)
#undef SIGMA_INST

}  // namespace sigma
