// a3w — op-level selective scan backward for WIDE states: 16 < d_state <= 256, padded to NP = 32, 64, 128, 256
// (scan_op_npad), any batch / dim / groups / L, contiguous (batch, dim, L) and (batch, G, N, L) operands, fp32 / fp16 / bf16
// read and written natively.  Every entry point (sigma_scan_bwd, _split, _det) runs it for d_state > 16: it is deterministic
// by construction, with no float atomic anywhere (dB / dC / dA / dD / ddelta_bias leave as partials, summed in a fixed order by
// sum_parts_det_kernel).
//
// Why not more instances of scan_op_bwd.cu: that kernel keeps h for a whole 32-position tile in shared memory (32 positions x NP
// states x 32 channels), 172 KB at NP = 32 and more than an SM has beyond.  Here h is never stashed for a whole tile.
//
// Three launches after the state sweep (the generic forward with `hs`: the state at the start of every 32-position tile):
// (1) scan_op_bwd_wide_kernel.  A CTA owns 32 channels of one (batch, group) — ONE PER LANE — and a chunk of SC = min(NP, 64)
//     states — warp w the SPT = 8 states [8w, 8w + 8) of the chunk.  Per 32-position tile, walked backwards:
//       * a forward pass from the tile-start state writes a checkpoint every 4 positions (thread-private shared memory);
//       * each 4-position sub-tile, last first, recomputes its four states into registers from its checkpoint, then runs the
//         reverse recurrence  dh_l = a_{l+1}·dh_{l+1} + dout_l·C_l  over them (bwd_kernel.cuh:173-227's arithmetic);
//       * dB / dC of a position are a sum over the 32 channels = the 32 lanes: one transpose_reduce of the 16 values (8 states
//         x {B, C}) per warp, no shared-memory traffic; the CTA's sums go to partials per channel tile of a group;
//       * du and the ddelta terms (sums over the states) are summed over the warps through shared memory once per sub-tile in
//         warp order, and leave as fp32 partials per state chunk;
//       * dA accumulates per thread (per tile, then across tiles) and leaves as a partial per batch.
//     Each thread pays three ex2 per (state, position) — checkpoint pass, sub-tile recompute, reverse step — instead of the
//     stash kernel's two.
// (2) scan_op_bwd_wide_finish_kernel: one warp per (batch, channel) row sums the state-chunk partials, adds dout·D, applies the
//     softplus derivative, writes du / ddelta in the element type, and leaves the row's dD / ddelta_bias partial.
// (3) sum_parts_det_kernel: dB / dC over the channel tiles of a group, dA / dD / ddelta_bias over the batch.
#include <algorithm>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "scan_core.cuh"

namespace sigma {

constexpr int WD_LT = 32;                 // positions per tile: the spacing of the state sweep's checkpoints `hs`
constexpr int WD_SUB = 4;                 // positions per sub-tile, recomputed into registers
constexpr int WD_NSUB = WD_LT / WD_SUB;   // checkpoints per tile
constexpr int WD_DT = 32;                 // channels per CTA, one per lane
constexpr int WD_SPT = 8;                 // states per thread
constexpr int WD_P = 33;                  // pitch of the [row][position] tiles: lanes reading one position of 32 rows hit 32 banks

struct ScanBwdWideParams {
  const void *u, *delta, *B, *C, *dout;   // element type T
  const float *A, *D, *bias, *hs;
  void *du, *ddelta;                      // element type T
  float *part_du, *part_X;   // (nsc, batch, dim, L): per state chunk, sum over its states of dh·delta'·B / of the ddelta terms
  float *part_B, *part_C;    // (tiles_per_group, batch, G, N, L)
  float *part_dA;            // (batch, dim, N)
  float *part_dD, *part_db;  // (batch, dim)
  int batch, dim, L, N, G, dpg, tiles_per_group, ntiles, nsc, softplus;
};

__host__ __device__ constexpr int wide_warps(int NP) { return (NP < 64 ? NP : 64) / WD_SPT; }

__host__ __device__ constexpr int wide_smem_floats(int NP) {
  // u, delta', dout (32 rows, du / X overwrite u / dout), B, C (SC rows, dB / dC overwrite them), the per-warp du / X slots of
  // a sub-tile (two buffers), the checkpoints (NSUB x SPT per thread)
  return 3 * WD_DT * WD_P + 2 * (8 * wide_warps(NP)) * WD_P + 2 * wide_warps(NP) * 2 * WD_SUB * 32 +
         WD_NSUB * WD_SPT * 32 * wide_warps(NP);
}

template <typename T, int NP>
__global__ void __launch_bounds__(32 * wide_warps(NP), 2) scan_op_bwd_wide_kernel(const ScanBwdWideParams p) {
  constexpr int W = wide_warps(NP), SC = 8 * W, NTH = 32 * W, SPT = WD_SPT;
  const T *pu = (const T *)p.u, *pdl = (const T *)p.delta, *pdo = (const T *)p.dout, *pB = (const T *)p.B, *pC = (const T *)p.C;
  extern __shared__ __align__(16) float smem[];
  float *sU = smem, *sDl = sU + WD_DT * WD_P, *sDo = sDl + WD_DT * WD_P;   // [channel][position]
  float *sB = sDo + WD_DT * WD_P, *sC = sB + SC * WD_P;                   // [state of the chunk][position]
  float *sSlot = sC + SC * WD_P;                                          // [buffer][warp][du | X][sub-tile position][channel]
  float *sCk = sSlot + 2 * W * 2 * WD_SUB * 32;                           // [checkpoint][s][thread]

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int g = blockIdx.x / p.tiles_per_group, tg = blockIdx.x - g * p.tiles_per_group;
  const int d_in_g0 = tg * WD_DT, d0 = g * p.dpg + d_in_g0;
  const int nch = min(WD_DT, p.dpg - d_in_g0);
  const bool ch_ok = lane < nch;
  const int d = d0 + (ch_ok ? lane : 0);
  const int sc = blockIdx.y, n0 = sc * SC + warp * SPT;   // this thread's first state
  const int b = blockIdx.z;
  const long long row0 = ((long long)b * p.dim + d0) * p.L;          // contiguous (batch, dim, L)
  const long long bc0 = ((long long)b * p.G + g) * p.N * (long long)p.L;

  float a2[SPT], Araw[SPT], dh[SPT], dAacc[SPT];
#pragma unroll
  for (int s = 0; s < SPT; ++s) {
    const int n = n0 + s;
    Araw[s] = (ch_ok && n < p.N) ? p.A[(long long)d * p.N + n] : 0.f;
    a2[s] = Araw[s] * kLog2e;
    dh[s] = 0.f;
    dAacc[s] = 0.f;
  }

  for (int t = p.ntiles - 1; t >= 0; --t) {
    const int l0 = t * WD_LT, npos = min(WD_LT, p.L - l0);
    // ---- load the tile: u, delta, dout rows of the 32 channels, B / C rows of the chunk's states (zero outside) ----
    for (int i = tid; i < (3 * WD_DT + 2 * SC) * WD_LT; i += NTH) {
      const int row = i >> 5, e = i & 31;
      float v = 0.f;
      if (e < npos) {
        if (row < WD_DT) { if (row < nch) v = to_f32(pu[row0 + (long long)row * p.L + l0 + e]); }
        else if (row < 2 * WD_DT) { if (row - WD_DT < nch) v = to_f32(pdl[row0 + (long long)(row - WD_DT) * p.L + l0 + e]); }
        else if (row < 3 * WD_DT) { if (row - 2 * WD_DT < nch) v = to_f32(pdo[row0 + (long long)(row - 2 * WD_DT) * p.L + l0 + e]); }
        else if (row < 3 * WD_DT + SC) { const int n = sc * SC + row - 3 * WD_DT; if (n < p.N) v = to_f32(pB[bc0 + (long long)n * p.L + l0 + e]); }
        else { const int n = sc * SC + row - 3 * WD_DT - SC; if (n < p.N) v = to_f32(pC[bc0 + (long long)n * p.L + l0 + e]); }
      }
      smem[row * WD_P + e] = v;
    }
    __syncthreads();
    // delta' once per (channel, position), in place; zero outside the valid channels and positions
    for (int i = tid; i < WD_DT * WD_LT; i += NTH) {
      const int c = i >> 5, e = i & 31;
      if (c < nch && e < npos) {
        const float raw = sDl[c * WD_P + e] + (p.bias ? p.bias[d0 + c] : 0.f);
        sDl[c * WD_P + e] = p.softplus ? softplus20(raw) : raw;
      }
    }
    __syncthreads();

    // ---- checkpoint pass: the state before every 4-position sub-tile, from the tile-start state ----
    {
      float h[SPT];
      const float *hs_row = p.hs + (((long long)b * p.dim + d) * p.ntiles + t) * NP + n0;
#pragma unroll
      for (int s = 0; s < SPT; ++s) h[s] = ch_ok ? hs_row[s] : 0.f;
      for (int k = 0; k < WD_NSUB && WD_SUB * k < npos; ++k) {
#pragma unroll
        for (int s = 0; s < SPT; ++s) sCk[(k * SPT + s) * NTH + tid] = h[s];
        if (WD_SUB * (k + 1) >= npos) break;
#pragma unroll
        for (int j = 0; j < WD_SUB; ++j) {
          const int i = WD_SUB * k + j;
          const float dl = sDl[lane * WD_P + i];
          const float dlu = dl * sU[lane * WD_P + i];
#pragma unroll
          for (int s = 0; s < SPT; ++s) h[s] = fmaf(ex2(dl * a2[s]), h[s], dlu * sB[(warp * SPT + s) * WD_P + i]);
        }
      }
    }

    // ---- reverse walk, one sub-tile at a time (dA: per-tile partial sums folded into the running total) ----
    float dAt[SPT];
#pragma unroll
    for (int s = 0; s < SPT; ++s) dAt[s] = 0.f;
    for (int k = (npos - 1) / WD_SUB; k >= 0; --k) {
      float hsub[WD_SUB][SPT];
      {
        float h[SPT];
#pragma unroll
        for (int s = 0; s < SPT; ++s) h[s] = sCk[(k * SPT + s) * NTH + tid];
#pragma unroll
        for (int j = 0; j < WD_SUB; ++j) {
          const int i = WD_SUB * k + j;
          if (i < npos) {
            const float dl = sDl[lane * WD_P + i];
            const float dlu = dl * sU[lane * WD_P + i];
#pragma unroll
            for (int s = 0; s < SPT; ++s) h[s] = fmaf(ex2(dl * a2[s]), h[s], dlu * sB[(warp * SPT + s) * WD_P + i]);
          }
#pragma unroll
          for (int s = 0; s < SPT; ++s) hsub[j][s] = h[s];
        }
      }
      float *slot = sSlot + (k & 1) * W * 2 * WD_SUB * 32;
#pragma unroll
      for (int j = WD_SUB - 1; j >= 0; --j) {
        const int i = WD_SUB * k + j;
        if (i >= npos) continue;
        const float dl = sDl[lane * WD_P + i];
        const float ui = sU[lane * WD_P + i];
        const float dy = sDo[lane * WD_P + i];
        float ddl = 0.f, dui = 0.f;
        float cBC[2 * SPT];   // [0, SPT): dB contributions, [SPT, 2 SPT): dC
#pragma unroll
        for (int s = 0; s < SPT; ++s) {
          const float Bn = sB[(warp * SPT + s) * WD_P + i], Cn = sC[(warp * SPT + s) * WD_P + i];
          const float hi = hsub[j][s];
          const float hprev = j > 0 ? hsub[j > 0 ? j - 1 : 0][s] : sCk[(k * SPT + s) * NTH + tid];
          const float a = ex2(dl * a2[s]);
          dh[s] = fmaf(dy, Cn, dh[s]);                 // gradient reaching h_i (bwd_kernel.cuh:173-199)
          cBC[SPT + s] = dy * hi;                       // dC contribution (:225)
          const float da = dh[s] * hprev;               // d/da of a·h_{i-1}
          ddl = fmaf(da * a, Araw[s], fmaf(dh[s] * Bn, ui, ddl));   // (:206)
          dAt[s] = fmaf(da * a, dl, dAt[s]);            // (:208)
          cBC[s] = dh[s] * dl * ui;                     // dB contribution (:224)
          dui = fmaf(dh[s] * dl, Bn, dui);              // (:205)
          dh[s] *= a;
        }
        // dB / dC of position i: the sum over the 32 channels (lanes); lane pairs (2m, 2m+1) end with value `which`
        int which = 0;
        const float v = transpose_reduce<2 * SPT, 16>(cBC, lane, which);
        // every lane has read B / C at position i (the shuffles above consumed them): overwrite them with dB / dC in place
        if ((lane & 1) == 0) (which < SPT ? sB : sC)[(warp * SPT + (which & (SPT - 1))) * WD_P + i] = v;
        slot[((warp * 2 + 0) * WD_SUB + j) * 32 + lane] = dui;
        slot[((warp * 2 + 1) * WD_SUB + j) * 32 + lane] = ddl;
      }
      __syncthreads();
      // du / X of the sub-tile: the warps' sums in warp order, into the u / dout rows (no longer read at these positions);
      // the slot buffer alternates, so the next sub-tile's writes need no second barrier
      for (int idx = tid; idx < 2 * WD_SUB * 32; idx += NTH) {
        const int which = idx / (WD_SUB * 32), j = (idx >> 5) % WD_SUB, c = idx & 31, i = WD_SUB * k + j;
        float v = 0.f;
#pragma unroll
        for (int w = 0; w < W; ++w) v += slot[((w * 2 + which) * WD_SUB + j) * 32 + c];
        if (i < npos) (which ? sDo : sU)[c * WD_P + i] = v;
      }
    }
#pragma unroll
    for (int s = 0; s < SPT; ++s) dAacc[s] += dAt[s];
    __syncthreads();
    // ---- write the tile's partials: du / X rows per state chunk, dB / dC rows per channel tile ----
    for (int i = tid; i < 2 * WD_DT * WD_LT; i += NTH) {
      const int which = i / (WD_DT * WD_LT), r = (i >> 5) % WD_DT, e = i & 31;
      if (r < nch && e < npos) {
        const long long o = (long long)sc * p.batch * p.dim * p.L + row0 + (long long)r * p.L + l0 + e;
        (which ? p.part_X : p.part_du)[o] = (which ? sDo : sU)[r * WD_P + e];
      }
    }
    for (int i = tid; i < 2 * SC * WD_LT; i += NTH) {
      const int which = i / (SC * WD_LT), r = (i >> 5) % SC, e = i & 31, n = sc * SC + r;
      if (n < p.N && e < npos) {
        const long long o = (long long)tg * p.batch * p.G * p.N * p.L + bc0 + (long long)n * p.L + l0 + e;
        (which ? p.part_C : p.part_B)[o] = (which ? sC : sB)[r * WD_P + e];
      }
    }
    __syncthreads();
  }
  if (ch_ok) {
    const long long bd = (long long)b * p.dim + d;
#pragma unroll
    for (int s = 0; s < SPT; ++s)
      if (n0 + s < p.N) p.part_dA[bd * p.N + n0 + s] = dAacc[s];
  }
}

// One warp per (batch, channel) row: du = dout·D + the chunks' du, ddelta = softplus'(raw)·(the chunks' X), in the element type;
// the row's dD / ddelta_bias partials (lane sums, then a fixed butterfly).
template <typename T>
__global__ void __launch_bounds__(256) scan_op_bwd_wide_finish_kernel(const ScanBwdWideParams p) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (long long)p.batch * p.dim) return;
  const int d = (int)(row % p.dim);
  const T *pu = (const T *)p.u, *pdl = (const T *)p.delta, *pdo = (const T *)p.dout;
  T *du = (T *)p.du, *dd = (T *)p.ddelta;
  const float bias = p.bias ? p.bias[d] : 0.f, Dv = p.D ? p.D[d] : 0.f;
  const long long chunk = (long long)p.batch * p.dim * p.L;
  float dDacc = 0.f, dbacc = 0.f;
  for (int l = lane; l < p.L; l += 32) {
    const long long o = row * p.L + l;
    float dui = 0.f, X = 0.f;
    for (int c = 0; c < p.nsc; ++c) {
      dui += p.part_du[c * chunk + o];
      X += p.part_X[c * chunk + o];
    }
    const float dy = to_f32(pdo[o]), ui = to_f32(pu[o]);
    const float raw = to_f32(pdl[o]) + bias;
    dui = fmaf(dy, Dv, dui);                                                          // (:143,250)
    dDacc = fmaf(dy, ui, dDacc);                                                      // (:144)
    if (p.softplus && raw <= 20.f) X *= __fdividef(1.f, 1.f + ex2(-raw * kLog2e));   // (:241-245)
    dbacc += X;
    du[o] = from_f32<T>(dui);
    dd[o] = from_f32<T>(X);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    dDacc += __shfl_xor_sync(0xffffffffu, dDacc, off);
    dbacc += __shfl_xor_sync(0xffffffffu, dbacc, off);
  }
  if (lane == 0) {
    p.part_dD[row] = dDacc;
    p.part_db[row] = dbacc;
  }
}

static size_t wide_tpg(int dim, int G) { return (size_t)(dim / G + WD_DT - 1) / WD_DT; }
static int wide_nsc(int NP) { return NP / (8 * wide_warps(NP)); }

// workspace: [hs (batch, dim, ntiles, NP)] [du / X partials (nsc, batch, dim, L) each] [dB / dC partials (tiles_per_group, batch,
// G, N, L) each] [dA partials (batch, dim, N)] [dD / ddelta_bias partials (batch, dim) each]
size_t scan_op_bwd_wide_workspace_bytes(int batch, int dim, int L, int N, int G) {
  if (batch <= 0 || dim <= 0 || L <= 0 || N <= 16 || N > 256 || G <= 0 || dim % G) return 0;
  const int NP = scan_op_npad(N);
  const size_t ntiles = (L + WD_LT - 1) / WD_LT, bdl = (size_t)batch * dim * L;
  return align256((size_t)batch * dim * ntiles * NP * sizeof(float)) + 2 * align256(wide_nsc(NP) * bdl * sizeof(float)) +
         2 * align256(wide_tpg(dim, G) * batch * G * N * L * sizeof(float)) + align256((size_t)batch * dim * N * sizeof(float)) +
         2 * align256((size_t)batch * dim * sizeof(float));
}

ScanOpPlan scan_op_bwd_wide_plan(int L) {
  ScanOpPlan pl;
  pl.ntiles = (L + WD_LT - 1) / WD_LT;
  pl.nsplit = 1;
  pl.tiles_per_split = pl.ntiles;
  pl.DT = WD_DT;
  pl.nst = 1;
  return pl;
}

template <typename T, int NP>
static int launch_bwd_wide(const ScanBwdWideParams &p, cudaStream_t stream) {
  const size_t smem = (size_t)wide_smem_floats(NP) * sizeof(float);
  SIGMA_CHECK_CUDA(cudaFuncSetAttribute(scan_op_bwd_wide_kernel<T, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(p.G * p.tiles_per_group, p.nsc, p.batch);
  scan_op_bwd_wide_kernel<T, NP><<<grid, 32 * wide_warps(NP), smem, stream>>>(p);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

// all tensors contiguous, element type T; deterministic whichever entry point calls it
template <typename T>
int scan_op_bwd_wide(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D, const float *bias,
                     const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC, float *dD, float *dbias, int batch,
                     int dim, int L, int N, int G, int softplus, void *ws, size_t ws_bytes, cudaStream_t stream) {
  const size_t need = scan_op_bwd_wide_workspace_bytes(batch, dim, L, N, G);
  if (need == 0) { set_error("sigma_scan_bwd: bad wide-state call (d_state=%d)", N); return SIGMA_EINVAL; }
  if (ws == nullptr || ws_bytes < need) {
    set_error("sigma_scan_bwd: workspace too small (%zu < %zu)", ws_bytes, need);
    return SIGMA_EWORKSPACE;
  }
  const int NP = scan_op_npad(N);
  ScanBwdWideParams p;
  p.u = u; p.delta = delta; p.B = B; p.C = C; p.dout = dout; p.A = A; p.D = D; p.bias = bias; p.du = du; p.ddelta = ddelta;
  p.batch = batch; p.dim = dim; p.L = L; p.N = N; p.G = G; p.dpg = dim / G;
  p.tiles_per_group = (int)wide_tpg(dim, G);
  p.ntiles = (L + WD_LT - 1) / WD_LT;
  p.nsc = wide_nsc(NP);
  p.softplus = softplus;
  const size_t bdl = (size_t)batch * dim * L;
  const size_t hs_b = align256((size_t)batch * dim * p.ntiles * NP * sizeof(float));
  const size_t x_b = align256(p.nsc * bdl * sizeof(float));
  const size_t bc_b = align256((size_t)p.tiles_per_group * batch * G * N * L * sizeof(float));
  const size_t da_b = align256((size_t)batch * dim * N * sizeof(float)), dd_b = align256((size_t)batch * dim * sizeof(float));
  char *w = (char *)ws;
  float *hs = (float *)w;
  p.hs = hs;
  p.part_du = (float *)(w + hs_b);
  p.part_X = (float *)(w + hs_b + x_b);
  p.part_B = (float *)(w + hs_b + 2 * x_b);
  p.part_C = (float *)(w + hs_b + 2 * x_b + bc_b);
  p.part_dA = (float *)(w + hs_b + 2 * x_b + 2 * bc_b);
  p.part_dD = (float *)(w + hs_b + 2 * x_b + 2 * bc_b + da_b);
  p.part_db = (float *)(w + hs_b + 2 * x_b + 2 * bc_b + da_b + dd_b);

  // state sweep: the generic forward leaves the tile-start states in hs; its output lands in du, overwritten below
  sigma_scan_strides st;
  st.u_batch = st.delta_batch = st.out_batch = (int64_t)dim * L;
  st.u_dim = st.delta_dim = st.out_dim = L;
  st.A_dim = N; st.A_dstate = 1;
  st.B_batch = st.C_batch = (int64_t)G * N * L;
  st.B_group = st.C_group = (int64_t)N * L;
  st.B_dstate = st.C_dstate = L;
  int rc = scan_op_fwd_generic<T>(u, delta, A, B, C, D, bias, du, nullptr, hs, batch, dim, L, N, G, softplus, st, nullptr, 0, 1, stream);
  if (rc) return rc;
  switch (NP) {
    case 32: rc = launch_bwd_wide<T, 32>(p, stream); break;
    case 64: rc = launch_bwd_wide<T, 64>(p, stream); break;
    case 128: rc = launch_bwd_wide<T, 128>(p, stream); break;
    default: rc = launch_bwd_wide<T, 256>(p, stream); break;
  }
  if (rc) return rc;
  const long long rows = (long long)batch * dim;
  scan_op_bwd_wide_finish_kernel<T><<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>(p);
  SIGMA_CHECK_LAUNCH();
  // fixed-order sums: dB / dC over the channel tiles of a group, dA / dD / ddelta_bias over the batch
  const long long bgnl = (long long)batch * G * N * L, dn = (long long)dim * N;
  if ((rc = sum_parts_det_launch(p.part_B, p.tiles_per_group, bgnl, bgnl, 0, dB, stream))) return rc;
  if ((rc = sum_parts_det_launch(p.part_C, p.tiles_per_group, bgnl, bgnl, 0, dC, stream))) return rc;
  if ((rc = sum_parts_det_launch(p.part_dA, batch, dn, dn, 0, dA, stream))) return rc;
  if (dD && (rc = sum_parts_det_launch(p.part_dD, batch, dim, dim, 0, dD, stream))) return rc;
  if (dbias && (rc = sum_parts_det_launch(p.part_db, batch, dim, dim, 0, dbias, stream))) return rc;
  return SIGMA_OK;
}

#define SIGMA_INST(T)                                                                                                             \
  template int scan_op_bwd_wide<T>(const void *, const void *, const float *, const void *, const void *, const float *,         \
                                   const float *, const void *, void *, void *, float *, float *, float *, float *, float *, int, \
                                   int, int, int, int, int, void *, size_t, cudaStream_t);
SIGMA_INST(float)
SIGMA_INST(__half)
SIGMA_INST(__nv_bfloat16)
#undef SIGMA_INST

}  // namespace sigma
