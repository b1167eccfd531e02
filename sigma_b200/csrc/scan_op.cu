// a1 — op-level selective scan forward, GENERIC path: any strides / ragged rows / any d_state <= 256 / channel groups
// that are not a multiple of 32.  Shapes TMA can express (every Sigma call) take scan_op_tma.cu instead.
// (reference: csrc/selective_scan/selective_scan.cpp:165-249, selective_scan_fwd_kernel.cuh:64-206).
// fp16 / bf16 are read and written natively (converted on the way into / out of shared memory; all arithmetic fp32).
//
// Layout is the reference's: u/delta/out (B, KD, L) and B/C (B, G, N, L), L contiguous.  A CTA owns
// 32 channels of one (batch, group) and walks L in tiles of 32 positions; tiles are staged in
// shared memory with cp.async (double buffered, [row][position] with a 36-float pitch so that both
// the channel-major reads and the 16-byte copies are bank-conflict free), the recurrence runs out
// of registers (scan_core.cuh), and the y tile goes back through shared memory so global stores
// are 128-byte rows.  When batch·KD cannot fill the GPU the sequence is cut into segments:
// MODE_SUMMARY computes each segment's (prod a, h_end) from h=0, a tiny combine kernel chains
// them, MODE_APPLY redoes the segment from its true start state and writes out.
#include <algorithm>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "scan_core.cuh"

namespace sigma {

constexpr int OP_LT = 32;   // positions per tile
constexpr int OP_LTP = 36;  // smem row pitch (floats)
constexpr int OP_DT = 32;   // channels per CTA
constexpr int OP_NST = 2;   // cp.async stages

struct ScanOpParams {
  const void *u, *delta, *B, *C;   // element type T of the kernel instantiation
  const float *A, *D, *bias;
  void *out;
  float *x, *carry;
  float *hs;  // optional: state at the START of every 32-position tile, (batch, dim, ntiles, NP) — consumed by the backward
  int batch, dim, L, N, G, dpg, tiles_per_group;
  int softplus;
  long long u_b, u_d, dl_b, dl_d, A_d, A_n, B_b, B_g, B_n, C_b, C_g, C_n, o_b, o_d;
  int nsplit, tiles_per_split, ntiles, nchunks;
  int vec_in, vec_out;
};

__host__ __device__ constexpr int op_smem_floats(int NP) {
  return OP_NST * (2 * OP_DT + 2 * NP) * OP_LTP + OP_DT * OP_LTP;
}

template <typename T, int SPT, int LPC, int MODE>
__global__ void __launch_bounds__(32 * LPC) scan_op_kernel(const ScanOpParams p) {
  constexpr bool F32 = sizeof(T) == 4;
  constexpr int NP = SPT * LPC;        // padded state count
  constexpr int CPW = 32 / LPC;        // channels per warp
  constexpr int NTHREADS = 32 * LPC;   // OP_DT / CPW warps
  constexpr int STAGE_ROWS = 2 * OP_DT + 2 * NP;
  constexpr bool WITH_Y = MODE != MODE_SUMMARY;

  extern __shared__ __align__(16) float smem[];
  float *sY = smem + OP_NST * STAGE_ROWS * OP_LTP;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q = lane % LPC;
  const int c_local = warp * CPW + lane / LPC;
  const int g = blockIdx.x / p.tiles_per_group;
  const int tg = blockIdx.x - g * p.tiles_per_group;
  const int d_in_g0 = tg * OP_DT;
  const int d0 = g * p.dpg + d_in_g0;              // first channel of this CTA
  const int nch = min(OP_DT, p.dpg - d_in_g0);     // valid channels in this CTA
  const bool ch_ok = c_local < nch;
  const int d = d0 + (ch_ok ? c_local : 0);
  const int b = blockIdx.z;
  const int split = blockIdx.y;
  const int t0 = split * p.tiles_per_split;
  const int t1 = min(p.ntiles, t0 + p.tiles_per_split);

  const T *gu = (const T *)p.u + (long long)b * p.u_b + (long long)d0 * p.u_d;
  const T *gdl = (const T *)p.delta + (long long)b * p.dl_b + (long long)d0 * p.dl_d;
  const T *gB = (const T *)p.B + (long long)b * p.B_b + (long long)g * p.B_g;
  const T *gC = (const T *)p.C + (long long)b * p.C_b + (long long)g * p.C_g;

  // --- per-thread constants ---
  float a2[SPT], h[SPT];
#pragma unroll
  for (int s = 0; s < SPT; ++s) {
    const int n = q * SPT + s;
    a2[s] = (ch_ok && n < p.N) ? p.A[(long long)d * p.A_d + (long long)n * p.A_n] * kLog2e : 0.f;
    h[s] = 0.f;
  }
  float *carry_row = nullptr;
  if (MODE != MODE_SERIAL) {
    carry_row = p.carry + (((long long)b * p.dim + d) * p.nsplit + split) * 2 * NP;
    if (MODE == MODE_APPLY && ch_ok) {
#pragma unroll
      for (int s = 0; s < SPT; ++s) h[s] = carry_row[NP + q * SPT + s];
    }
  }
  const float bias = (p.bias && ch_ok) ? p.bias[d] : 0.f;
  const float Dv = (p.D && ch_ok) ? p.D[d] : 0.f;
  float sumdl = 0.f;  // Σ delta' since the start of this CTA's walk (per channel, identical on its LPC lanes)

  // --- tile loader: rows [0,32) u, [32,64) delta, [64,64+NP) B, [64+NP,64+2NP) C ---
  auto load_tile = [&](int t, int st) {
    float *sbase = smem + st * STAGE_ROWS * OP_LTP;
    const int l0 = t * OP_LT;
    constexpr int ROWS = WITH_Y ? STAGE_ROWS : (2 * OP_DT + NP);
    if (F32 && p.vec_in) {
      for (int i = tid; i < ROWS * (OP_LT / 4); i += NTHREADS) {
        const int row = i >> 3, ck = i & 7;
        const int l = l0 + ck * 4;
        const T *src;
        bool ok;
        if (row < OP_DT) { ok = row < nch; src = gu + (long long)row * p.u_d; }
        else if (row < 2 * OP_DT) { ok = (row - OP_DT) < nch; src = gdl + (long long)(row - OP_DT) * p.dl_d; }
        else if (row < 2 * OP_DT + NP) { const int n = row - 2 * OP_DT; ok = n < p.N; src = gB + (long long)n * p.B_n; }
        else { const int n = row - 2 * OP_DT - NP; ok = n < p.N; src = gC + (long long)n * p.C_n; }
        int nb = ok ? min(4, p.L - l) * 4 : 0;
        nb = max(nb, 0);
        if constexpr (F32) cp_async16(sbase + row * OP_LTP + ck * 4, nb > 0 ? (const void *)(src + l) : (const void *)p.u, nb);
      }
    } else {
      for (int i = tid; i < ROWS * OP_LT; i += NTHREADS) {
        const int row = i >> 5, e = i & 31;
        const int l = l0 + e;
        const T *src;
        bool ok;
        if (row < OP_DT) { ok = row < nch; src = gu + (long long)row * p.u_d; }
        else if (row < 2 * OP_DT) { ok = (row - OP_DT) < nch; src = gdl + (long long)(row - OP_DT) * p.dl_d; }
        else if (row < 2 * OP_DT + NP) { const int n = row - 2 * OP_DT; ok = n < p.N; src = gB + (long long)n * p.B_n; }
        else { const int n = row - 2 * OP_DT - NP; ok = n < p.N; src = gC + (long long)n * p.C_n; }
        ok = ok && l < p.L;
        if constexpr (F32) cp_async4(sbase + row * OP_LTP + e, ok ? (const void *)(src + l) : (const void *)p.u, ok ? 4 : 0);
        else sbase[row * OP_LTP + e] = ok ? to_f32(src[l]) : 0.f;   // 16-bit elements: plain load, widened on the way in
      }
    }
  };

  if (t0 < t1) load_tile(t0, 0);
  cp_async_commit();

  for (int t = t0; t < t1; ++t) {
    const int st = (t - t0) & 1;
    if (t + 1 < t1) load_tile(t + 1, st ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();

    if (MODE == MODE_SERIAL && p.hs != nullptr && ch_ok) {
      float *hrow = p.hs + (((long long)b * p.dim + d) * p.ntiles + t) * NP + q * SPT;
#pragma unroll
      for (int s = 0; s < SPT; ++s) hrow[s] = h[s];
    }
    const float *sU = smem + st * STAGE_ROWS * OP_LTP;
    const float *sDl = sU + OP_DT * OP_LTP;
    const float *sB = sDl + OP_DT * OP_LTP;
    const float *sC = sB + NP * OP_LTP;
    const int npos = min(OP_LT, p.L - t * OP_LT);

#pragma unroll 1
    for (int j = 0; j < OP_LT / 4; ++j) {
      const int cnt = npos - 4 * j;
      if (cnt <= 0) break;
      const float4 u4 = *reinterpret_cast<const float4 *>(sU + c_local * OP_LTP + 4 * j);
      const float4 r4 = *reinterpret_cast<const float4 *>(sDl + c_local * OP_LTP + 4 * j);
      float raw[4] = {r4.x + bias, r4.y + bias, r4.z + bias, r4.w + bias};
      float dl[4];
      shared_softplus4<LPC>(raw, p.softplus != 0, lane, dl);
      constexpr bool VEC_BC = SPT <= 4;  // wide SPT (N > 16) reads B/C per position to bound registers
      float4 Bv[VEC_BC ? SPT : 1], Cv[VEC_BC ? SPT : 1];
      if (VEC_BC) {
#pragma unroll
        for (int s = 0; s < (VEC_BC ? SPT : 1); ++s) {
          Bv[s] = *reinterpret_cast<const float4 *>(sB + (q * SPT + s) * OP_LTP + 4 * j);
          if (WITH_Y) Cv[s] = *reinterpret_cast<const float4 *>(sC + (q * SPT + s) * OP_LTP + 4 * j);
        }
      }
      float y[4] = {0.f, 0.f, 0.f, 0.f};
      const float uu[4] = {u4.x, u4.y, u4.z, u4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i < cnt) {
          float Bs[SPT], Cs[SPT];
#pragma unroll
          for (int s = 0; s < SPT; ++s) {
            if (VEC_BC) {
              Bs[s] = f4_get(Bv[VEC_BC ? s : 0], i);
              Cs[s] = WITH_Y ? f4_get(Cv[VEC_BC ? s : 0], i) : 0.f;
            } else {
              Bs[s] = sB[(q * SPT + s) * OP_LTP + 4 * j + i];
              Cs[s] = WITH_Y ? sC[(q * SPT + s) * OP_LTP + 4 * j + i] : 0.f;
            }
          }
          scan_step<SPT, WITH_Y>(h, a2, dl[i], uu[i], Bs, Cs, y[i]);
          sumdl += dl[i];
        }
      }
      if (WITH_Y) {
#pragma unroll
        for (int i = 0; i < 4; ++i) y[i] = channel_reduce<LPC>(y[i]);
        if (q == 0) {
          float4 o;
          o.x = fmaf(Dv, uu[0], y[0]); o.y = fmaf(Dv, uu[1], y[1]);
          o.z = fmaf(Dv, uu[2], y[2]); o.w = fmaf(Dv, uu[3], y[3]);
          *reinterpret_cast<float4 *>(sY + c_local * OP_LTP + 4 * j) = o;
        }
      }
    }

    if (WITH_Y) {
      __syncwarp();
      // this warp's CPW rows of the y tile -> global, 128-byte rows
      T *go = (T *)p.out + (long long)b * p.o_b + (long long)d0 * p.o_d + (long long)t * OP_LT;
      if (F32 && p.vec_out) {
        for (int i = lane; i < CPW * (OP_LT / 4); i += 32) {
          const int r = warp * CPW + (i >> 3), ck = i & 7;
          if (r < nch && 4 * ck < npos) {
            const float4 v = *reinterpret_cast<const float4 *>(sY + r * OP_LTP + 4 * ck);
            float *dst = (float *)go + (long long)r * p.o_d + 4 * ck;
            if (4 * ck + 4 <= npos) *reinterpret_cast<float4 *>(dst) = v;
            else {
              dst[0] = v.x;
              if (4 * ck + 1 < npos) dst[1] = v.y;
              if (4 * ck + 2 < npos) dst[2] = v.z;
            }
          }
        }
      } else {
        for (int rr = 0; rr < CPW; ++rr) {
          const int r = warp * CPW + rr;
          if (r < nch && lane < npos) go[(long long)r * p.o_d + lane] = from_f32<T>(sY[r * OP_LTP + lane]);
        }
      }
      // x checkpoints: (prod a, h) at the end of every 2048-chunk (selective_scan_fwd_kernel.cuh:181-184)
      if (p.x != nullptr) {
        const int lend = t * OP_LT + npos;
        if ((lend & 2047) == 0 || lend == p.L) {
          if (ch_ok) {
            const int c = (lend - 1) >> 11;
            float *xr = p.x + (((long long)b * p.dim + d) * p.nchunks + c) * 2 * p.N;
#pragma unroll
            for (int s = 0; s < SPT; ++s) {
              const int n = q * SPT + s;
              if (n < p.N) {   // (prod a since the SEQUENCE start, h): SSMScanPrefixCallbackOp's running prefix
                float P = ex2(a2[s] * sumdl);
                if (MODE == MODE_APPLY) P *= carry_row[q * SPT + s];
                xr[2 * n] = P;
                xr[2 * n + 1] = h[s];
              }
            }
          }
        }
      }
    }
    __syncthreads();  // stage st may be overwritten by the prefetch issued next iteration
  }
  cp_async_wait<0>();

  if (MODE == MODE_SUMMARY && ch_ok) {
#pragma unroll
    for (int s = 0; s < SPT; ++s) {
      carry_row[q * SPT + s] = ex2(a2[s] * sumdl);
      carry_row[NP + q * SPT + s] = h[s];
    }
  }
}

// carry[row][split] = (P, h_local_end) -> (product of P over the PRECEDING segments, H_start):
// H_0 = 0, H_{s+1} = P_s·H_s + h_s.  (The prefix product feeds the running-prefix component of the chunk states `x`.)
__global__ void scan_combine_kernel(float *carry, long long nrows, int nsplit, int NP) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= nrows * NP) return;
  const long long row = idx / NP;
  const int n = (int)(idx - row * NP);
  float H = 0.f, Pc = 1.f;
  float *base = carry + row * nsplit * 2 * NP + n;
  // eight segments at a time: their 16 loads are issued together (the walk is in place, so a plain loop serialises on one
  // L2 round trip per segment: 14 us for 24 segments at batch 1)
  for (int s0 = 0; s0 < nsplit; s0 += 8) {
    float P[8], hl[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool in = s0 + j < nsplit;
      P[j] = in ? base[(long long)(s0 + j) * 2 * NP] : 1.f;
      hl[j] = in ? base[(long long)(s0 + j) * 2 * NP + NP] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (s0 + j < nsplit) {
        base[(long long)(s0 + j) * 2 * NP] = Pc;
        base[(long long)(s0 + j) * 2 * NP + NP] = H;
        H = fmaf(P[j], H, hl[j]);
        Pc *= P[j];
      }
    }
  }
}

// ---- host side ----
static int pick_npad(int N) {
  if (N <= 4) return 4;
  if (N <= 8) return 8;
  if (N <= 16) return 16;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  if (N <= 128) return 128;
  return 256;
}

template <typename T, int SPT, int LPC>
static int launch_scan_op(ScanOpParams &p, cudaStream_t stream) {
  constexpr int NP = SPT * LPC;
  const size_t smem = (size_t)op_smem_floats(NP) * sizeof(float);
  dim3 grid(p.G * p.tiles_per_group, p.nsplit, p.batch);
  dim3 block(32 * LPC);
  auto set_attr = [&](const void *fn) -> cudaError_t {
    return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  };
  if (p.nsplit == 1) {
    SIGMA_CHECK_CUDA(set_attr((const void *)scan_op_kernel<T, SPT, LPC, MODE_SERIAL>));
    scan_op_kernel<T, SPT, LPC, MODE_SERIAL><<<grid, block, smem, stream>>>(p);
    SIGMA_CHECK_LAUNCH();
  } else {
    SIGMA_CHECK_CUDA(set_attr((const void *)scan_op_kernel<T, SPT, LPC, MODE_SUMMARY>));
    SIGMA_CHECK_CUDA(set_attr((const void *)scan_op_kernel<T, SPT, LPC, MODE_APPLY>));
    scan_op_kernel<T, SPT, LPC, MODE_SUMMARY><<<grid, block, smem, stream>>>(p);
    SIGMA_CHECK_LAUNCH();
    const long long nrows = (long long)p.batch * p.dim;
    const long long tot = nrows * NP;
    scan_combine_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, stream>>>(p.carry, nrows, p.nsplit, NP);
    SIGMA_CHECK_LAUNCH();
    scan_op_kernel<T, SPT, LPC, MODE_APPLY><<<grid, block, smem, stream>>>(p);
    SIGMA_CHECK_LAUNCH();
  }
  return SIGMA_OK;
}

constexpr int kGenMaxSplit = 64;   // the carry workspace holds this many segments per row (scan_op_workspace_bytes)

// lanes per channel: d_state > 16 runs with up to 16 lanes per channel (8-16 states per lane) so that no instantiation spills
static int pick_lpc(int NP) { return NP <= 4 ? 1 : (NP <= 8 ? 2 : (NP <= 32 ? 4 : (NP <= 128 ? NP / 8 : 16))); }

// Decide how many L-segments to use.  Splitting doubles the exp work, so only do it when the
// unsplit grid leaves most of the SMs idle.  A forced count is capped like the automatic one.
ScanOpPlan scan_op_fwd_generic_plan(int batch, int dim, int L, int N, int G, bool have_ws, int force_split) {
  ScanOpPlan pl;
  pl.ntiles = (L + OP_LT - 1) / OP_LT;
  pl.DT = OP_DT;
  pl.nst = OP_NST;
  const long long warps = (long long)batch * G * ((dim / G + OP_DT - 1) / OP_DT) * pick_lpc(pick_npad(N));
  int nsplit = 1;
  const long long target = kNumSMs * 8;  // warps for a reasonably busy machine
  if (warps * 3 < target) nsplit = (int)std::min<long long>((target + warps - 1) / warps, kGenMaxSplit);
  if (force_split > 0) nsplit = std::min(force_split, kGenMaxSplit);
  if (!have_ws) nsplit = 1;
  int tps = (pl.ntiles + nsplit - 1) / nsplit;
  tps = std::max(tps, 1);
  nsplit = (pl.ntiles + tps - 1) / tps;
  pl.tiles_per_split = tps;
  pl.nsplit = std::max(nsplit, 1);
  return pl;
}

size_t scan_op_workspace_bytes(int batch, int dim, int dstate) {
  return (size_t)batch * dim * kGenMaxSplit * 2 * pick_npad(dstate) * sizeof(float);
}

int scan_op_npad(int N) { return pick_npad(N); }

// `hs` (nullable): state at the start of every 32-position tile, (batch, dim, ntiles, NP) — forces a single pass.
template <typename T>
int scan_op_fwd_generic(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                        const float *bias, void *out, float *x, float *hs, int batch, int dim, int L, int N, int G,
                        int softplus, const sigma_scan_strides &s, void *ws, size_t ws_bytes, int force_split,
                        cudaStream_t stream) {
  ScanOpParams p;
  p.hs = hs;
  if (hs != nullptr) force_split = 1;  // checkpoints are written by the serial walk only
  p.u = u; p.delta = delta; p.A = A; p.B = B; p.C = C; p.D = D; p.bias = bias;
  p.out = out; p.x = x; p.carry = (float *)ws;
  p.batch = batch; p.dim = dim; p.L = L; p.N = N; p.G = G; p.dpg = dim / G;
  p.tiles_per_group = (p.dpg + OP_DT - 1) / OP_DT;
  p.softplus = softplus;
  p.u_b = s.u_batch; p.u_d = s.u_dim; p.dl_b = s.delta_batch; p.dl_d = s.delta_dim;
  p.A_d = s.A_dim; p.A_n = s.A_dstate;
  p.B_b = s.B_batch; p.B_g = s.B_group; p.B_n = s.B_dstate;
  p.C_b = s.C_batch; p.C_g = s.C_group; p.C_n = s.C_dstate;
  p.o_b = s.out_batch; p.o_d = s.out_dim;
  p.nchunks = (L + 2047) / 2048;
  auto al16 = [](const void *ptr) { return ((uintptr_t)ptr & 15) == 0; };
  auto m4 = [](long long v) { return (v & 3) == 0; };
  p.vec_in = sizeof(T) == 4 && al16(u) && al16(delta) && al16(B) && al16(C) && m4(p.u_b) && m4(p.u_d) && m4(p.dl_b) &&
             m4(p.dl_d) && m4(p.B_b) && m4(p.B_g) && m4(p.B_n) && m4(p.C_b) && m4(p.C_g) && m4(p.C_n);
  p.vec_out = sizeof(T) == 4 && al16(out) && m4(p.o_b) && m4(p.o_d);

  const int NP = pick_npad(N);
  const bool have_ws = ws != nullptr && ws_bytes >= scan_op_workspace_bytes(batch, dim, N);
  const ScanOpPlan pl = scan_op_fwd_generic_plan(batch, dim, L, N, G, have_ws, force_split);
  p.ntiles = pl.ntiles;
  p.nsplit = pl.nsplit;
  p.tiles_per_split = pl.tiles_per_split;

  switch (NP) {
    case 4: return launch_scan_op<T, 4, 1>(p, stream);
    case 8: return launch_scan_op<T, 4, 2>(p, stream);
    case 16: return launch_scan_op<T, 4, 4>(p, stream);
    case 32: return launch_scan_op<T, 8, 4>(p, stream);
    case 64: return launch_scan_op<T, 8, 8>(p, stream);
    case 128: return launch_scan_op<T, 8, 16>(p, stream);
    default: return launch_scan_op<T, 16, 16>(p, stream);
  }
}

#define SIGMA_INST(T)                                                                                                       \
  template int scan_op_fwd_generic<T>(const void *, const void *, const float *, const void *, const void *, const float *, \
                                      const float *, void *, float *, float *, int, int, int, int, int, int,               \
                                      const sigma_scan_strides &, void *, size_t, int, cudaStream_t);
SIGMA_INST(float)
SIGMA_INST(__half)
SIGMA_INST(__nv_bfloat16)
#undef SIGMA_INST

}  // namespace sigma
