// Row-wise kernels of the channels-last pipeline:
//   row_norm_kernel  : [sum over K direction outputs] -> LayerNorm -> [· SiLU(z)] -> [· gate]   (one warp per row)
//                      = nn.LayerNorm (vmamba.py:1693,2173,...) when K=1, z=gate=NULL, and
//                      = CrossMerge sum + out_norm + y·SiLU(z) (vmamba.py:217-224,1077) otherwise;
//                      y / z fp32, bf16 or fp16, out fp32, bf16, fp16 or e4m3 rows (row_norm_launch lists the pairs)
//   layernorm_bwd    : dx, dgamma, dbeta of the LayerNorm, x / dy / dx fp32, bf16 or fp16
//   the e4m3 row quantizer and the decoder tail (bilinear x2 + LayerNorm [+ head], pooling, scale-add), fp32
// All are HBM-bound; loads/stores are 16-byte (8 for 16-bit, 4 for e4m3 elements), rows are contiguous in the channel dimension.
// gamma, beta, gate and all arithmetic are fp32.
#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace sigma {


__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// (x - mean)·rstd·gamma + beta [· SiLU(z)] [· gate] of float4 idx of a row: the arithmetic of the stores below, for the e4m3
// instances, which hold the whole row before they store it
__device__ __forceinline__ float4 norm_gate4(float4 x, float mean, float rstd, const RowNormParams &p, int idx, float4 z, bool has_z,
                                             const float *gate_row) {
  const float4 g = __ldg(reinterpret_cast<const float4 *>(p.gamma) + idx);
  const float4 b = __ldg(reinterpret_cast<const float4 *>(p.beta) + idx);
  float4 o;
  o.x = fmaf((x.x - mean) * rstd, g.x, b.x);
  o.y = fmaf((x.y - mean) * rstd, g.y, b.y);
  o.z = fmaf((x.z - mean) * rstd, g.z, b.z);
  o.w = fmaf((x.w - mean) * rstd, g.w, b.w);
  if (has_z) { o.x *= silu(z.x); o.y *= silu(z.y); o.z *= silu(z.z); o.w *= silu(z.w); }
  if (gate_row) {
    const float4 gg = __ldg(reinterpret_cast<const float4 *>(gate_row) + idx);
    o.x *= gg.x; o.y *= gg.y; o.z *= gg.z; o.w *= gg.w;
  }
  return o;
}

// TI: element type of y and z, TO: of out (row_norm_launch's ti / to; E4M3Rows: e4m3 bytes + p.qscale); gamma, beta, gate and
// all arithmetic are fp32
template <int MAXV, typename TI, typename TO>
__global__ void __launch_bounds__(256) row_norm_kernel(const RowNormParams p) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= p.rows) return;
  const long long bi = row / p.rows_per_batch, ri = row - bi * p.rows_per_batch;
  const TI *in = reinterpret_cast<const TI *>(p.y) + bi * p.in_batch_stride + ri * p.D;
  const int nvec = p.D >> 2;
  float4 x[MAXV];
  float s = 0.f;
#pragma unroll
  for (int v = 0; v < MAXV; ++v) {
    const int idx = lane + 32 * v;
    x[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (idx < nvec) {
      float4 a = ld4g(in + 4 * idx);
      for (int k = 1; k < p.K; ++k) {
        const float4 b = ld4g(in + k * p.k_stride + 4 * idx);
        a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
      }
      x[v] = a;
      s += (a.x + a.y) + (a.z + a.w);
    }
  }
  const float mean = warp_sum(s) / (float)p.D;
  float q = 0.f;
#pragma unroll
  for (int v = 0; v < MAXV; ++v) {
    if (lane + 32 * v < nvec) {
      const float dx = x[v].x - mean, dy = x[v].y - mean, dz = x[v].z - mean, dw = x[v].w - mean;
      q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)p.D + p.eps);
  TO *out = reinterpret_cast<TO *>(p.out) + bi * p.out_batch_stride + ri * p.out_row_stride;
  const TI *zr = p.z ? reinterpret_cast<const TI *>(p.z) + row * p.z_row_stride : nullptr;
  const float *gr = p.gate ? p.gate + bi * p.D : nullptr;
  if constexpr (std::is_same<TO, E4M3Rows>::value) {   // the whole row first (its amax sets the scale), then e4m3
    float am = 0.f;
#pragma unroll
    for (int v = 0; v < MAXV; ++v) {
      const int idx = lane + 32 * v;
      if (idx < nvec) {
        x[v] = norm_gate4(x[v], mean, rstd, p, idx, zr ? ld4g(zr + 4 * idx) : make_float4(0.f, 0.f, 0.f, 0.f), zr != nullptr, gr);
        am = fmaxf(am, amax4(x[v]));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
    const float inv = e4m3_inv_scale(am);
#pragma unroll
    for (int v = 0; v < MAXV; ++v) {
      const int idx = lane + 32 * v;
      if (idx < nvec) reinterpret_cast<uint32_t *>(out)[idx] = e4m3x4(x[v], inv);
    }
    if (lane == 0) p.qscale[row] = e4m3_scale(am);
  } else {
#pragma unroll
  for (int v = 0; v < MAXV; ++v) {
    const int idx = lane + 32 * v;
    if (idx < nvec) {
      const float4 g = __ldg(reinterpret_cast<const float4 *>(p.gamma) + idx);
      const float4 b = __ldg(reinterpret_cast<const float4 *>(p.beta) + idx);
      float4 o;
      o.x = fmaf((x[v].x - mean) * rstd, g.x, b.x);
      o.y = fmaf((x[v].y - mean) * rstd, g.y, b.y);
      o.z = fmaf((x[v].z - mean) * rstd, g.z, b.z);
      o.w = fmaf((x[v].w - mean) * rstd, g.w, b.w);
      if (zr) {
        const float4 zz = ld4g(zr + 4 * idx);
        o.x *= silu(zz.x); o.y *= silu(zz.y); o.z *= silu(zz.z); o.w *= silu(zz.w);
      }
      if (gr) {
        const float4 gg = __ldg(reinterpret_cast<const float4 *>(gr) + idx);
        o.x *= gg.x; o.y *= gg.y; o.z *= gg.z; o.w *= gg.w;
      }
      st4(out + 4 * idx, o);
    }
  }
  }
}

// Fast path for the row lengths the models use (D/4 = LPR·V float4 with LPR in {8,16,32} lanes per row):
// a warp works on 32/LPR rows at once, every lane issues all its K·V (+V for z) 16-byte loads before the first use
// (the generic kernel above has one load in flight per lane inside a runtime-K loop: ~45 % of HBM peak under ncu),
// reductions are LPR-wide shuffles.  y and z are dead after this kernel: streaming loads (evict-first).
template <int LPR, int V, int K, int MODE, typename TI, typename TO>
__global__ void __launch_bounds__(256) row_norm_fast_kernel(const RowNormParams p) {
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, sub = lane / LPR, l = lane % LPR;
  const long long row_raw = ((long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + sub;
  const bool valid = row_raw < p.rows;
  const long long row = valid ? row_raw : p.rows - 1;     // keep the warp convergent for the shuffles
  long long bi = 0, ri = row;
  if (p.rows_per_batch < p.rows) { bi = row / p.rows_per_batch; ri = row - bi * p.rows_per_batch; }   // 64-bit division only when batched
  const TI *in = reinterpret_cast<const TI *>(p.y) + bi * p.in_batch_stride + ri * p.D;
  float4 x[V], kk[K > 1 ? (K - 1) * V : 1], zz[V];
  if (MODE == 1) {
    // gather the 2x2 pixel block of output row (b, i, j); quadrant q of the row = pixel (2i + (q&1), 2j + (q>>1))
    const int H2 = (p.gH + 1) >> 1, W2 = (p.gW + 1) >> 1, cq = (p.D >> 2) >> 2;   // float4 per source pixel
    const long long b = row / ((long long)H2 * W2);
    const int rem = (int)(row - b * H2 * W2), i = rem / W2, j = rem - i * W2;
    const TI *src = reinterpret_cast<const TI *>(p.y) + b * p.gH * p.gW * 4 * cq;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int idx = l + LPR * v, q = idx / cq, c4 = idx - q * cq;
      const int hh = 2 * i + (q & 1), ww = 2 * j + (q >> 1);
      x[v] = (hh < p.gH && ww < p.gW) ? ld4g(src + 4 * (((long long)hh * p.gW + ww) * cq + c4)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else {
#pragma unroll
    for (int v = 0; v < V; ++v) x[v] = ld4cs(in + 4 * (l + LPR * v));
  }
#pragma unroll
  for (int k = 1; k < K; ++k)
#pragma unroll
    for (int v = 0; v < V; ++v) kk[(k - 1) * V + v] = ld4cs(in + k * p.k_stride + 4 * (l + LPR * v));
  const bool has_z = p.z != nullptr;
  if (has_z) {
    const TI *zr = reinterpret_cast<const TI *>(p.z) + row * p.z_row_stride;
#pragma unroll
    for (int v = 0; v < V; ++v) zz[v] = ld4cs(zr + 4 * (l + LPR * v));
  }
  float s = 0.f;
#pragma unroll
  for (int v = 0; v < V; ++v) {
#pragma unroll
    for (int k = 1; k < K; ++k) {
      const float4 b = kk[(k - 1) * V + v];
      x[v].x += b.x; x[v].y += b.y; x[v].z += b.z; x[v].w += b.w;
    }
    s += (x[v].x + x[v].y) + (x[v].z + x[v].w);
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)p.D;
  float q = 0.f;
#pragma unroll
  for (int v = 0; v < V; ++v) {
    const float dx = x[v].x - mean, dy = x[v].y - mean, dz = x[v].z - mean, dw = x[v].w - mean;
    q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)p.D + p.eps);
  TO *out = reinterpret_cast<TO *>(p.out) + bi * p.out_batch_stride + ri * p.out_row_stride;
  if (MODE == 2) {
    const int p2 = (int)(row & 1), p1 = (int)((row >> 1) & 1);
    const long long pix = row >> 2, b = pix / ((long long)p.gH * p.gW);
    const int rem = (int)(pix - b * p.gH * p.gW), h = rem / p.gW, w = rem - h * p.gW;
    out = reinterpret_cast<TO *>(p.out) + (((b * 2 * p.gH + 2 * h + p1) * 2 * p.gW) + 2 * w + p2) * p.D;
  }
  const float4 *gr = p.gate ? reinterpret_cast<const float4 *>(p.gate + bi * p.D) : nullptr;
  if constexpr (std::is_same<TO, E4M3Rows>::value) {   // the whole row first (its amax sets the scale), then e4m3
    float am = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      x[v] = norm_gate4(x[v], mean, rstd, p, l + LPR * v, zz[v], has_z, reinterpret_cast<const float *>(gr));
      am = fmaxf(am, amax4(x[v]));
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
    const float inv = e4m3_inv_scale(am);
    if (valid) {
#pragma unroll
      for (int v = 0; v < V; ++v) reinterpret_cast<uint32_t *>(out)[l + LPR * v] = e4m3x4(x[v], inv);
      if (l == 0) p.qscale[row] = e4m3_scale(am);
    }
  } else {
#pragma unroll
  for (int v = 0; v < V; ++v) {
    const int idx = l + LPR * v;
    const float4 g = __ldg(reinterpret_cast<const float4 *>(p.gamma) + idx);
    const float4 b = __ldg(reinterpret_cast<const float4 *>(p.beta) + idx);
    float4 o;
    o.x = fmaf((x[v].x - mean) * rstd, g.x, b.x);
    o.y = fmaf((x[v].y - mean) * rstd, g.y, b.y);
    o.z = fmaf((x[v].z - mean) * rstd, g.z, b.z);
    o.w = fmaf((x[v].w - mean) * rstd, g.w, b.w);
    if (has_z) { o.x *= silu(zz[v].x); o.y *= silu(zz[v].y); o.z *= silu(zz[v].z); o.w *= silu(zz[v].w); }
    if (gr) {
      const float4 gg = __ldg(gr + idx);
      o.x *= gg.x; o.y *= gg.y; o.z *= gg.z; o.w *= gg.w;
    }
    if (valid) st4(out + 4 * idx, o);
  }
  }
}

// ---- row_norm_launch: one dispatcher over the element pairs (TI, TO) ----
// What each pair has instances for:
//  * fast kernel, plain rows (mode 0): K = 1 for every pair; K = 2 and 4 (the direction merge of a scan output) where the input
//    is 16-bit or both types are fp32.  Patch-merge gather (mode 1): fp32 input, K = 1.  Pixel shuffle (mode 2): fp32 only, K = 1.
//  * generic kernel, plain rows only: D <= 4096, or D <= 1024 for e4m3 output, which holds the whole row in registers before it
//    stores it (a wider row would spill).
//  * e4m3 output: K = 1 or 4 only.
template <typename TI, typename TO>
struct RowNormPair {
  static constexpr bool E4M3 = std::is_same<TO, E4M3Rows>::value;
  static constexpr bool F32_IN = std::is_same<TI, float>::value, F32_OUT = std::is_same<TO, float>::value;
  static constexpr int GENERIC_MAXV = E4M3 ? 8 : 32;
  static constexpr bool k_ok(int K) { return !E4M3 || K == 1 || K == 4; }
  static constexpr bool fast(int mode, int K) {
    if (mode == 0) return K == 1 || ((!F32_IN || F32_OUT) && (K == 2 || K == 4) && k_ok(K));
    return K == 1 && F32_IN && (mode == 1 || (mode == 2 && F32_OUT));
  }
};

template <int LPR, int V, int K, int MODE, typename TI, typename TO>
static bool row_norm_fast_if(const RowNormParams &p, unsigned grid, cudaStream_t stream) {
  if constexpr (RowNormPair<TI, TO>::fast(MODE, K)) {
    if (p.mode == MODE && p.K == K) {
      row_norm_fast_kernel<LPR, V, K, MODE, TI, TO><<<grid, 256, 0, stream>>>(p);
      return true;
    }
  }
  return false;
}

template <typename TI, typename TO, int LPR, int V>
static bool row_norm_fast_k(const RowNormParams &p, cudaStream_t stream) {
  const int rows_per_cta = 8 * (32 / LPR);   // 8 warps
  const unsigned grid = (unsigned)((p.rows + rows_per_cta - 1) / rows_per_cta);
  return row_norm_fast_if<LPR, V, 1, 0, TI, TO>(p, grid, stream) || row_norm_fast_if<LPR, V, 2, 0, TI, TO>(p, grid, stream) ||
         row_norm_fast_if<LPR, V, 4, 0, TI, TO>(p, grid, stream) || row_norm_fast_if<LPR, V, 1, 1, TI, TO>(p, grid, stream) ||
         row_norm_fast_if<LPR, V, 1, 2, TI, TO>(p, grid, stream);
}

// picks (lanes per row, float4 per lane) for D; false if D, a stride or (mode, K) has no fast instance
template <typename TI, typename TO>
static bool row_norm_fast(const RowNormParams &p, cudaStream_t stream) {
  if ((p.D & 3) || (p.k_stride & 3) || (p.in_batch_stride & 3) || (p.out_row_stride & 3) || (p.out_batch_stride & 3) ||
      (p.z_row_stride & 3))
    return false;
  const int nvec = p.D >> 2;
#define TRY(LPR, V) if (nvec == (LPR) * (V)) return row_norm_fast_k<TI, TO, LPR, V>(p, stream)
  TRY(8, 2); TRY(8, 3); TRY(8, 4);
  TRY(16, 3); TRY(16, 4);
  TRY(32, 3); TRY(32, 4); TRY(32, 6); TRY(32, 8); TRY(32, 12); TRY(32, 16);
#undef TRY
  return false;
}

// the generic kernel with the fewest float4 slots (1, 2, 4, ... GENERIC_MAXV) that hold nvec
template <typename TI, typename TO, int MAXV = 1>
static void row_norm_generic(const RowNormParams &p, int nvec, cudaStream_t stream) {
  if constexpr (MAXV < RowNormPair<TI, TO>::GENERIC_MAXV) {
    if (nvec > 32 * MAXV) return row_norm_generic<TI, TO, 2 * MAXV>(p, nvec, stream);
  }
  row_norm_kernel<MAXV, TI, TO><<<(unsigned)((p.rows + 7) / 8), 256, 0, stream>>>(p);
}

template <typename TI, typename TO>
static int row_norm_dispatch(const RowNormParams &p, cudaStream_t stream) {
  using Pair = RowNormPair<TI, TO>;
  if (p.rows == 0) return SIGMA_OK;
  if (!row_norm_fast<TI, TO>(p, stream)) {
    const int nvec = p.D >> 2;
    if (p.mode != 0 || !Pair::k_ok(p.K) || nvec > 32 * Pair::GENERIC_MAXV) {
      set_error("row_norm: no instance for D=%d, mode %d, K=%d (gather / pixel-shuffle modes need D = 4·LPR·V; plain rows reach "
                "D <= %d%s)", p.D, p.mode, p.K, 128 * Pair::GENERIC_MAXV, Pair::E4M3 ? ", K = 1 or 4 for e4m3 output" : "");
      return SIGMA_EUNSUPPORTED;
    }
    row_norm_generic<TI, TO>(p, nvec, stream);
  }
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

int row_norm_launch(int ti, int to, const RowNormParams &p, cudaStream_t stream) {
  using bf16 = __nv_bfloat16;
  if (ti == SIGMA_F32 && to == SIGMA_F32) return row_norm_dispatch<float, float>(p, stream);
  if (ti == SIGMA_F32 && to == SIGMA_BF16) return row_norm_dispatch<float, bf16>(p, stream);
  if (ti == SIGMA_F32 && to == SIGMA_F16) return row_norm_dispatch<float, __half>(p, stream);
  if (ti == SIGMA_F32 && to == SIGMA_E4M3_ROWS) return row_norm_dispatch<float, E4M3Rows>(p, stream);
  if (ti == SIGMA_BF16 && to == SIGMA_BF16) return row_norm_dispatch<bf16, bf16>(p, stream);
  if (ti == SIGMA_BF16 && to == SIGMA_E4M3_ROWS) return row_norm_dispatch<bf16, E4M3Rows>(p, stream);
  if (ti == SIGMA_F16 && to == SIGMA_F16) return row_norm_dispatch<__half, __half>(p, stream);
  set_error("row_norm: no instances for element types (%d, %d)", ti, to);
  return SIGMA_EUNSUPPORTED;
}

// ---- standalone e4m3 row quantizer (the FP8 inference mode: weights per output channel, and activations no producer holds a
// row of): one warp per row, an amax pass and a quantizing pass over the row (the second one from L1 / L2) ----
template <typename TI>
__global__ void __launch_bounds__(256) quantize_e4m3_rows_kernel(const TI *__restrict__ x, long long ldx, unsigned char *__restrict__ q,
                                                                  long long ldq, float *__restrict__ scale, long long rows, int C) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const TI *xr = x + row * ldx;
  const int nvec = C >> 2;
  float am = 0.f;
  for (int i = lane; i < nvec; i += 32) am = fmaxf(am, amax4(ld4g(xr + 4 * i)));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
  const float inv = e4m3_inv_scale(am);
  uint32_t *qr = reinterpret_cast<uint32_t *>(q + row * ldq);
  for (int i = lane; i < nvec; i += 32) qr[i] = e4m3x4(ld4g(xr + 4 * i), inv);
  if (lane == 0) scale[row] = e4m3_scale(am);
}

int quantize_e4m3_rows_launch(const void *x, bool bf16, long long ldx, void *q, long long ldq, float *scale, long long rows, int C,
                              cudaStream_t stream) {
  if (rows == 0) return SIGMA_OK;
  const unsigned grid = (unsigned)((rows + 7) / 8);
  if (bf16)
    quantize_e4m3_rows_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>((const __nv_bfloat16 *)x, ldx, (unsigned char *)q, ldq, scale, rows, C);
  else
    quantize_e4m3_rows_kernel<float><<<grid, 256, 0, stream>>>((const float *)x, ldx, (unsigned char *)q, ldq, scale, rows, C);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

// ---- LayerNorm backward (training path): dx, dgamma, dbeta of y = (x - mean)·rstd·gamma + beta over the last dim ----
// Same lane layout as row_norm_fast_kernel (LPR lanes per row, V float4 per lane, 32/LPR rows per warp step); mean / rstd are
// recomputed from x (x is read anyway), so the forward saves nothing.  A warp walks rows with a grid stride and keeps its lanes'
// dgamma / dbeta columns in registers; they are reduced over the warp's sub-rows by shuffles and leave the warp as one
// atomicAdd per column (torch's GammaBetaBackwardCUDAKernel spent 5.9 ms per Sigma-tiny training step on this reduction).
// DET: instead of the atomics, warp w of the grid writes its column sums to part[w·D ...] (dgamma) and
// part[(nwarps + w)·D ...] (dbeta); sum_parts_det_kernel adds them in warp order.
// T: element type of x, dy and dx (float; __nv_bfloat16 / __half for bf16 / fp16 activations — gamma, the statistics, dgamma and
// dbeta stay fp32)
template <int LPR, int V, bool DET, typename T = float>
__device__ __forceinline__ void layernorm_bwd_body(const T *__restrict__ x, const T *__restrict__ dy, const float *__restrict__ gamma,
                                                   T *__restrict__ dx, float *__restrict__ dgamma, float *__restrict__ dbeta,
                                                   long long rows, int D, float eps, float *__restrict__ part) {
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane / LPR, l = lane % LPR;
  const long long wstride = (long long)gridDim.x * (blockDim.x >> 5);
  const float invD = 1.f / (float)D;
  constexpr bool GREG = V <= 6;        // wide rows re-read gamma through L1 instead of pinning 4·V more registers
  float4 g[GREG ? V : 1], dg[V], db[V];
  const float4 *gp = reinterpret_cast<const float4 *>(gamma) + l;
#pragma unroll
  for (int v = 0; v < V; ++v) {
    if (GREG) g[v] = __ldg(gp + LPR * v);
    dg[v] = make_float4(0.f, 0.f, 0.f, 0.f);
    db[v] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const long long nsteps = (rows + RPW - 1) / RPW;
  for (long long step = (long long)blockIdx.x * (blockDim.x >> 5) + warp; step < nsteps; step += wstride) {
    const long long row_raw = step * RPW + sub;
    const bool valid = row_raw < rows;
    const long long row = valid ? row_raw : rows - 1;
    float4 xv[V], dv[V];
    if constexpr (sizeof(T) == 4) {
      const float4 *xr = reinterpret_cast<const float4 *>(x + row * D), *dr = reinterpret_cast<const float4 *>(dy + row * D);
#pragma unroll
      for (int v = 0; v < V; ++v) { xv[v] = __ldcs(xr + l + LPR * v); dv[v] = __ldcs(dr + l + LPR * v); }
    } else {
      const T *xr = x + row * D, *dr = dy + row * D;
#pragma unroll
      for (int v = 0; v < V; ++v) { xv[v] = ld4cs(xr + 4 * (l + LPR * v)); dv[v] = ld4cs(dr + 4 * (l + LPR * v)); }
    }
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) s += (xv[v].x + xv[v].y) + (xv[v].z + xv[v].w);
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * invD;
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      xv[v].x -= mean; xv[v].y -= mean; xv[v].z -= mean; xv[v].w -= mean;
      q += (xv[v].x * xv[v].x + xv[v].y * xv[v].y) + (xv[v].z * xv[v].z + xv[v].w * xv[v].w);
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q * invD + eps);
    float s1 = 0.f, s2 = 0.f;          // Σ gamma·dy and Σ gamma·dy·xhat over the row
#pragma unroll
    for (int v = 0; v < V; ++v) {
      xv[v].x *= rstd; xv[v].y *= rstd; xv[v].z *= rstd; xv[v].w *= rstd;        // xhat
      const float4 gv = GREG ? g[GREG ? v : 0] : __ldg(gp + LPR * v);
      const float a0 = gv.x * dv[v].x, a1 = gv.y * dv[v].y, a2 = gv.z * dv[v].z, a3 = gv.w * dv[v].w;
      s1 += (a0 + a1) + (a2 + a3);
      s2 += (a0 * xv[v].x + a1 * xv[v].y) + (a2 * xv[v].z + a3 * xv[v].w);
    }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) {
      s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    }
    const float m1 = s1 * invD, m2 = s2 * invD;
    float4 *outr = reinterpret_cast<float4 *>(dx + row * D);   // bf16: only the row's address (st4 below)
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const float4 gv = GREG ? g[GREG ? v : 0] : __ldg(gp + LPR * v);
      float4 o;
      o.x = rstd * (gv.x * dv[v].x - m1 - xv[v].x * m2);
      o.y = rstd * (gv.y * dv[v].y - m1 - xv[v].y * m2);
      o.z = rstd * (gv.z * dv[v].z - m1 - xv[v].z * m2);
      o.w = rstd * (gv.w * dv[v].w - m1 - xv[v].w * m2);
      if (valid) {
        if constexpr (sizeof(T) == 4) outr[l + LPR * v] = o;
        else st4(dx + row * D + 4 * (l + LPR * v), o);
        dg[v].x = fmaf(dv[v].x, xv[v].x, dg[v].x); dg[v].y = fmaf(dv[v].y, xv[v].y, dg[v].y);
        dg[v].z = fmaf(dv[v].z, xv[v].z, dg[v].z); dg[v].w = fmaf(dv[v].w, xv[v].w, dg[v].w);
        db[v].x += dv[v].x; db[v].y += dv[v].y; db[v].z += dv[v].z; db[v].w += dv[v].w;
      }
    }
  }
  // the warp's sub-rows share columns: fold them onto sub-row 0
#pragma unroll
  for (int v = 0; v < V; ++v) {
#pragma unroll
    for (int o = LPR; o < 32; o <<= 1) {
      dg[v].x += __shfl_xor_sync(0xffffffffu, dg[v].x, o); dg[v].y += __shfl_xor_sync(0xffffffffu, dg[v].y, o);
      dg[v].z += __shfl_xor_sync(0xffffffffu, dg[v].z, o); dg[v].w += __shfl_xor_sync(0xffffffffu, dg[v].w, o);
      db[v].x += __shfl_xor_sync(0xffffffffu, db[v].x, o); db[v].y += __shfl_xor_sync(0xffffffffu, db[v].y, o);
      db[v].z += __shfl_xor_sync(0xffffffffu, db[v].z, o); db[v].w += __shfl_xor_sync(0xffffffffu, db[v].w, o);
    }
  }
  if (DET) {
    if (sub == 0) {
      const long long gw = (long long)blockIdx.x * (blockDim.x >> 5) + warp, nw = (long long)gridDim.x * (blockDim.x >> 5);
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int c = 4 * (l + LPR * v);
        *reinterpret_cast<float4 *>(part + gw * D + c) = dg[v];
        *reinterpret_cast<float4 *>(part + (nw + gw) * D + c) = db[v];
      }
    }
  } else if (sub == 0) {              // one red.global.add per column and warp (<= ~1M per call: the grid is sized for it)
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int c = 4 * (l + LPR * v);
      atomicAdd(dgamma + c, dg[v].x); atomicAdd(dgamma + c + 1, dg[v].y); atomicAdd(dgamma + c + 2, dg[v].z); atomicAdd(dgamma + c + 3, dg[v].w);
      atomicAdd(dbeta + c, db[v].x); atomicAdd(dbeta + c + 1, db[v].y); atomicAdd(dbeta + c + 2, db[v].z); atomicAdd(dbeta + c + 3, db[v].w);
    }
  }
}

template <int LPR, int V>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float *__restrict__ x, const float *__restrict__ dy,
                                                             const float *__restrict__ gamma, float *__restrict__ dx,
                                                             float *__restrict__ dgamma, float *__restrict__ dbeta, long long rows,
                                                             int D, float eps) {
  layernorm_bwd_body<LPR, V, false>(x, dy, gamma, dx, dgamma, dbeta, rows, D, eps, nullptr);
}

template <int LPR, int V>
__global__ void __launch_bounds__(256) layernorm_bwd_det_kernel(const float *__restrict__ x, const float *__restrict__ dy,
                                                                 const float *__restrict__ gamma, float *__restrict__ dx, long long rows,
                                                                 int D, float eps, float *__restrict__ part) {
  layernorm_bwd_body<LPR, V, true>(x, dy, gamma, dx, nullptr, nullptr, rows, D, eps, part);
}

template <int LPR, int V>
__global__ void __launch_bounds__(256) layernorm_bwd_bf16_kernel(const __nv_bfloat16 *__restrict__ x, const __nv_bfloat16 *__restrict__ dy,
                                                                  const float *__restrict__ gamma, __nv_bfloat16 *__restrict__ dx,
                                                                  float *__restrict__ dgamma, float *__restrict__ dbeta, long long rows,
                                                                  int D, float eps) {
  layernorm_bwd_body<LPR, V, false, __nv_bfloat16>(x, dy, gamma, dx, dgamma, dbeta, rows, D, eps, nullptr);
}

template <int LPR, int V>
__global__ void __launch_bounds__(256) layernorm_bwd_fp16_kernel(const __half *__restrict__ x, const __half *__restrict__ dy,
                                                                  const float *__restrict__ gamma, __half *__restrict__ dx,
                                                                  float *__restrict__ dgamma, float *__restrict__ dbeta, long long rows,
                                                                  int D, float eps) {
  layernorm_bwd_body<LPR, V, false, __half>(x, dy, gamma, dx, dgamma, dbeta, rows, D, eps, nullptr);
}

// enough CTAs to fill the machine, few enough that the 2·D atomics per warp stay negligible (a warp walks >= 4 steps);
// lanes per row as in the instantiation table of layernorm_bwd_launch
static unsigned layernorm_bwd_grid(long long rows, int D) {
  const int warps = 8, nvec = D >> 2, lpr = nvec % 32 == 0 && nvec >= 96 ? 32 : nvec % 16 == 0 && nvec >= 48 ? 16 : 8;
  const long long nsteps = (rows + 32 / lpr - 1) / (32 / lpr);
  return (unsigned)std::max<long long>(1, std::min<long long>(kNumSMs * 8, (nsteps + warps * 4 - 1) / (warps * 4)));
}

template <int LPR, int V>
static void layernorm_bwd_k(int dtype, const void *x, const void *dy, const float *gamma, void *dx, float *dgamma, float *dbeta,
                            long long rows, int D, float eps, float *part, cudaStream_t stream) {
  using bf = __nv_bfloat16;
  const int warps = 8;
  const unsigned grid = layernorm_bwd_grid(rows, D);
  if (dtype == SIGMA_F16) layernorm_bwd_fp16_kernel<LPR, V><<<grid, warps * 32, 0, stream>>>((const __half *)x, (const __half *)dy, gamma, (__half *)dx, dgamma, dbeta, rows, D, eps);
  else if (dtype == SIGMA_BF16) layernorm_bwd_bf16_kernel<LPR, V><<<grid, warps * 32, 0, stream>>>((const bf *)x, (const bf *)dy, gamma, (bf *)dx, dgamma, dbeta, rows, D, eps);
  else if (part) layernorm_bwd_det_kernel<LPR, V><<<grid, warps * 32, 0, stream>>>((const float *)x, (const float *)dy, gamma, (float *)dx, rows, D, eps, part);
  else layernorm_bwd_kernel<LPR, V><<<grid, warps * 32, 0, stream>>>((const float *)x, (const float *)dy, gamma, (float *)dx, dgamma, dbeta, rows, D, eps);
}

// deterministic build: one dgamma and one dbeta row of D floats per warp of the grid
size_t layernorm_bwd_det_workspace_bytes(long long rows, int D) {
  return (size_t)2 * layernorm_bwd_grid(rows, D) * 8 * D * sizeof(float);
}

// dgamma / dbeta are zeroed here and accumulated into; false if D has no instantiation (the fast forward's D set).
// part != nullptr: the deterministic build (layernorm_bwd_det_workspace_bytes of scratch), dgamma / dbeta written by the
// fixed-order sum over the grid's warps.  dtype: element type of x, dy and dx (SIGMA_BF16 / SIGMA_F16 never with part)
int layernorm_bwd_launch(int dtype, const void *x, const void *dy, const float *gamma, void *dx, float *dgamma, float *dbeta,
                         long long rows, int D, float eps, cudaStream_t stream, float *part) {
  if (D & 3) { set_error("layernorm_bwd: D=%d must be a multiple of 4", D); return SIGMA_EUNSUPPORTED; }
  if (rows == 0 && !part) return SIGMA_OK;
  if (rows == 0) {
    SIGMA_CHECK_CUDA(cudaMemsetAsync(dgamma, 0, (size_t)D * sizeof(float), stream));
    SIGMA_CHECK_CUDA(cudaMemsetAsync(dbeta, 0, (size_t)D * sizeof(float), stream));
    return SIGMA_OK;
  }
  if (!part) {
    SIGMA_CHECK_CUDA(cudaMemsetAsync(dgamma, 0, (size_t)D * sizeof(float), stream));
    SIGMA_CHECK_CUDA(cudaMemsetAsync(dbeta, 0, (size_t)D * sizeof(float), stream));
  }
  const int nvec = D >> 2;
  bool ok = false;
#define TRY(LPR, V) if (!ok && nvec == (LPR) * (V)) { layernorm_bwd_k<LPR, V>(dtype, x, dy, gamma, dx, dgamma, dbeta, rows, D, eps, part, stream); SIGMA_CHECK_LAUNCH(); ok = true; }
  TRY(8, 1) TRY(8, 2) TRY(8, 3) TRY(8, 4)
  TRY(16, 3) TRY(16, 4)
  TRY(32, 3) TRY(32, 4) TRY(32, 6) TRY(32, 8) TRY(32, 12)
#undef TRY
  if (!ok) {
    set_error("layernorm_bwd: D=%d has no instantiation (D/4 = lanes-per-row x vectors in {8x1..4, 16x3..4, 32x3,4,6,8,12})", D);
    return SIGMA_EUNSUPPORTED;
  }
  if (!part) return SIGMA_OK;
  const int nw = (int)layernorm_bwd_grid(rows, D) * 8;
  const int rc = sum_parts_det_launch(part, nw, D, D, 0, dgamma, stream);
  return rc ? rc : sum_parts_det_launch(part + (size_t)nw * D, nw, D, D, 0, dbeta, stream);
}

}  // namespace sigma

// =============================================================================================
// Decoder tail kernels (MambaDecoder.py:33-51, 76-97, 272-280; vmamba.py:1725-1757, 1800-1805)
// =============================================================================================
namespace sigma {

// F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) source taps for output index o:
// src = (o + 0.5)/2 - 0.5, clamped at 0 (PyTorch area_pixel_compute_source_index), i1 = min(i0+1, n-1)
__device__ __forceinline__ void bilinear2x_taps(int o, int n, int &i0, int &i1, float &w1) {
  float s = ((float)o + 0.5f) * 0.5f - 0.5f;
  s = fmaxf(s, 0.f);
  i0 = (int)s;
  i1 = min(i0 + 1, n - 1);
  w1 = s - (float)i0;
}

// out[b, oh, ow, :] = LayerNorm( bilinear2x(in)[b, oh, ow, :] ) — one warp per output pixel.
// With NCLS > 0 the normalised row is additionally projected by a (NCLS, C) matrix (the decoder's final
// 1x1 conv, MambaDecoder.py:279) and only the logits are written, in NCHW.
template <int MAXV, int NCLS>
__global__ void __launch_bounds__(256) upsample2x_norm_kernel(const float *__restrict__ in, const float *__restrict__ gamma,
                                                             const float *__restrict__ beta, const float *__restrict__ wcls,
                                                             float *__restrict__ out, int B, int Hin, int Win, int C,
                                                             float eps) {
  __shared__ float slog[NCLS > 0 ? NCLS : 1][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int Ho = 2 * Hin, Wo = 2 * Win;
  const long long npix = (long long)B * Ho * Wo;
  const int PPW = NCLS > 0 ? 4 : 1;  // pixels per warp
  const long long pix0 = ((long long)blockIdx.x * 8 + warp) * PPW;
  const int nvec = C >> 2;
  for (int pp = 0; pp < PPW; ++pp) {
    const long long pix = pix0 + pp;
    if (pix >= npix) break;
    const int b = (int)(pix / ((long long)Ho * Wo));
    const int rem = (int)(pix - (long long)b * Ho * Wo);
    const int oh = rem / Wo, ow = rem - oh * Wo;
    int h0, h1, w0, w1;
    float fh, fw;
    bilinear2x_taps(oh, Hin, h0, h1, fh);
    bilinear2x_taps(ow, Win, w0, w1, fw);
    const float c00 = (1.f - fh) * (1.f - fw), c01 = (1.f - fh) * fw, c10 = fh * (1.f - fw), c11 = fh * fw;
    const float *base = in + (long long)b * Hin * Win * C;
    const float4 *r00 = reinterpret_cast<const float4 *>(base + ((long long)h0 * Win + w0) * C);
    const float4 *r01 = reinterpret_cast<const float4 *>(base + ((long long)h0 * Win + w1) * C);
    const float4 *r10 = reinterpret_cast<const float4 *>(base + ((long long)h1 * Win + w0) * C);
    const float4 *r11 = reinterpret_cast<const float4 *>(base + ((long long)h1 * Win + w1) * C);
    float4 x[MAXV];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < MAXV; ++v) {
      const int idx = lane + 32 * v;
      x[v] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < nvec) {
        const float4 a = __ldg(r00 + idx), bq = __ldg(r01 + idx), c = __ldg(r10 + idx), d = __ldg(r11 + idx);
        // same association as PyTorch's upsample_bilinear2d: h0lambda*(w0l*a + w1l*b) + h1lambda*(w0l*c + w1l*d)
        x[v].x = (1.f - fh) * ((1.f - fw) * a.x + fw * bq.x) + fh * ((1.f - fw) * c.x + fw * d.x);
        x[v].y = (1.f - fh) * ((1.f - fw) * a.y + fw * bq.y) + fh * ((1.f - fw) * c.y + fw * d.y);
        x[v].z = (1.f - fh) * ((1.f - fw) * a.z + fw * bq.z) + fh * ((1.f - fw) * c.z + fw * d.z);
        x[v].w = (1.f - fh) * ((1.f - fw) * a.w + fw * bq.w) + fh * ((1.f - fw) * c.w + fw * d.w);
        s += (x[v].x + x[v].y) + (x[v].z + x[v].w);
      }
    }
    (void)c00; (void)c01; (void)c10; (void)c11;
    const float mean = warp_sum(s) / (float)C;
    float q = 0.f;
#pragma unroll
    for (int v = 0; v < MAXV; ++v)
      if (lane + 32 * v < nvec) {
        const float dx = x[v].x - mean, dy = x[v].y - mean, dz = x[v].z - mean, dw = x[v].w - mean;
        q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
    const float rstd = rsqrtf(warp_sum(q) / (float)C + eps);
    float acc[NCLS > 0 ? NCLS : 1];
#pragma unroll
    for (int c = 0; c < (NCLS > 0 ? NCLS : 1); ++c) acc[c] = 0.f;
#pragma unroll
    for (int v = 0; v < MAXV; ++v) {
      const int idx = lane + 32 * v;
      if (idx < nvec) {
        const float4 g = __ldg(reinterpret_cast<const float4 *>(gamma) + idx);
        const float4 bt = __ldg(reinterpret_cast<const float4 *>(beta) + idx);
        float4 o;
        o.x = fmaf((x[v].x - mean) * rstd, g.x, bt.x);
        o.y = fmaf((x[v].y - mean) * rstd, g.y, bt.y);
        o.z = fmaf((x[v].z - mean) * rstd, g.z, bt.z);
        o.w = fmaf((x[v].w - mean) * rstd, g.w, bt.w);
        if (NCLS > 0) {
#pragma unroll
          for (int c = 0; c < (NCLS > 0 ? NCLS : 1); ++c) {
            const float4 wv = __ldg(reinterpret_cast<const float4 *>(wcls + (long long)c * C) + idx);
            acc[c] = fmaf(o.x, wv.x, fmaf(o.y, wv.y, fmaf(o.z, wv.z, fmaf(o.w, wv.w, acc[c]))));
          }
        } else {
          reinterpret_cast<float4 *>(out + pix * C)[idx] = o;
        }
      }
    }
    if (NCLS > 0) {
#pragma unroll
      for (int c = 0; c < (NCLS > 0 ? NCLS : 1); ++c) {
        const float v = warp_sum(acc[c]);
        if (lane == 0) slog[c][warp * 4 + pp] = v;
      }
    }
  }
  if (NCLS > 0) {
    __syncthreads();
    // 32 consecutive pixels x NCLS classes -> NCHW, 128-byte runs per class
    const long long p0 = (long long)blockIdx.x * 32;
    const long long HWo = (long long)Ho * Wo;
    for (int i = threadIdx.x; i < NCLS * 32; i += blockDim.x) {
      const int c = i >> 5, j = i & 31;
      const long long pix = p0 + j;
      if (pix < npix) {
        const long long b = pix / HWo, r = pix - b * HWo;
        out[(b * NCLS + c) * HWo + r] = slog[c][j];
      }
    }
  }
}

// ---- plain bilinear x2 (no norm), channels-last: one thread per (output pixel, 4 channels) ----
__global__ void __launch_bounds__(256) upsample2x_plain_kernel(const float *__restrict__ in, float *__restrict__ out, int B,
                                                              int Hin, int Win, int C) {
  // thread = (output pixel, 4 channels); grid.y = image, so all index math is 32-bit (no 64-bit divisions)
  const unsigned nvec = C >> 2, Ho = 2 * Hin, Wo = 2 * Win, per_img = Ho * Wo * nvec;
  const int b = blockIdx.y;
  const float4 *src = reinterpret_cast<const float4 *>(in) + (long long)b * Hin * Win * nvec;
  float4 *dst = reinterpret_cast<float4 *>(out) + (long long)b * per_img;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < per_img; i += gridDim.x * blockDim.x) {
    const unsigned pix = i / nvec, q = i - pix * nvec;
    const unsigned oh = pix / Wo, ow = pix - oh * Wo;
    int h0, h1, w0, w1;
    float fh, fw;
    bilinear2x_taps((int)oh, Hin, h0, h1, fh);
    bilinear2x_taps((int)ow, Win, w0, w1, fw);
    const float4 *base = src + q;
    const float4 a = __ldg(base + (unsigned)(h0 * Win + w0) * nvec), bq = __ldg(base + (unsigned)(h0 * Win + w1) * nvec);
    const float4 c = __ldg(base + (unsigned)(h1 * Win + w0) * nvec), d = __ldg(base + (unsigned)(h1 * Win + w1) * nvec);
    float4 o;   // same association as PyTorch's upsample_bilinear2d
    o.x = (1.f - fh) * ((1.f - fw) * a.x + fw * bq.x) + fh * ((1.f - fw) * c.x + fw * d.x);
    o.y = (1.f - fh) * ((1.f - fw) * a.y + fw * bq.y) + fh * ((1.f - fw) * c.y + fw * d.y);
    o.z = (1.f - fh) * ((1.f - fw) * a.z + fw * bq.z) + fh * ((1.f - fw) * c.z + fw * d.z);
    o.w = (1.f - fh) * ((1.f - fw) * a.w + fw * bq.w) + fh * ((1.f - fw) * c.w + fw * d.w);
    dst[i] = o;
  }
}

// ---- bilinear x2 -> LayerNorm -> (NCLS, C) head, for C = 4·LPR·V: a warp works on 32/LPR output pixels at once
// (LPR lanes per pixel, V float4 per lane), so LayerNorm and the NCLS dot products reduce with log2(LPR) shuffles
// for 32/LPR pixels instead of 5 per pixel; the head weights are read from shared memory (LDS.128, 128-byte rows).
// The generic kernel above spends 55 warp shuffles per pixel: 5 ms for 32 x 480 x 640 pixels. ----
// CTA = an 8 x 32 tile of OUTPUT pixels.  Its (8/2 + 2) x (32/2 + 2) input pixels are staged ONCE in shared memory:
// bilinear x2 reads every input pixel for 16 (tap, output pixel) pairs, and with the taps read from global memory
// the kernel was bound by L2 -> L1 traffic (~17 GB for 74 images; 5.0 ms).  Warp w owns output row w of the tile:
// 32 consecutive pixels, 32/LPR x PX = 8 per pass.
constexpr int UH_TH = 8, UH_TW = 32, UH_IH = UH_TH / 2 + 2, UH_IW = UH_TW / 2 + 2;

template <int LPR, int V, int NCLS>
__global__ void __launch_bounds__(256) upsample2x_norm_head_fast_kernel(const float *__restrict__ in, const float *__restrict__ gamma,
                                                                        const float *__restrict__ beta, const float *__restrict__ wcls,
                                                                        float *__restrict__ out, int B, int Hin, int Win, float eps) {
  constexpr int RPW = 32 / LPR, PX = 2, C4 = LPR * V, C = 4 * C4, PASSES = 32 / (RPW * PX);
  extern __shared__ __align__(16) float smem_uh[];
  float4 *tile = reinterpret_cast<float4 *>(smem_uh);                         // [UH_IH][UH_IW][C4]
  float *sw = smem_uh + UH_IH * UH_IW * C;                                    // [NCLS][C]
  float *slog = sw + NCLS * C;                                                // [8][NCLS][32]
  const int Ho = 2 * Hin, Wo = 2 * Win;
  const int b = blockIdx.z, oh_t = blockIdx.y * UH_TH, ow_t = blockIdx.x * UH_TW;
  const int i0 = oh_t / 2 - 1, j0 = ow_t / 2 - 1;                             // input coordinates of tile[0][0]
  const float4 *src = reinterpret_cast<const float4 *>(in + (long long)b * Hin * Win * C);
  for (int i = threadIdx.x; i < UH_IH * UH_IW * C4; i += blockDim.x) {
    const int pix = i / C4, q = i - pix * C4, ri = pix / UH_IW, ci = pix - ri * UH_IW;
    const int hh = min(max(i0 + ri, 0), Hin - 1), ww = min(max(j0 + ci, 0), Win - 1);   // edge replicate = the taps' clamping
    tile[i] = __ldg(src + ((long long)hh * Win + ww) * C4 + q);
  }
  for (int i = threadIdx.x; i < NCLS * C; i += blockDim.x) sw[i] = wcls[i];
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, sub = lane / LPR, l = lane % LPR;
  const int oh = oh_t + warp;
  if (oh >= Ho) return;                                                        // warp-uniform; no CTA barrier below
  int h0, h1;
  float fh;
  bilinear2x_taps(oh, Hin, h0, h1, fh);
  const float4 *row0 = tile + (h0 - i0) * UH_IW * C4 + l, *row1 = tile + (h1 - i0) * UH_IW * C4 + l;
  float4 g[V], bt[V];
#pragma unroll
  for (int v = 0; v < V; ++v) {
    g[v] = __ldg(reinterpret_cast<const float4 *>(gamma) + l + LPR * v);
    bt[v] = __ldg(reinterpret_cast<const float4 *>(beta) + l + LPR * v);
  }
  float *mylog = slog + warp * NCLS * 32;
#pragma unroll 1
  for (int pass = 0; pass < PASSES; ++pass) {
    float4 x[PX][V];
    float mean[PX], rstd[PX];
#pragma unroll
    for (int px = 0; px < PX; ++px) {
      const int ow = min(ow_t + (pass * PX + px) * RPW + sub, Wo - 1);         // past the right edge: recompute the last column
      int w0, w1;
      float fw;
      bilinear2x_taps(ow, Win, w0, w1, fw);
      const int c0 = (w0 - j0) * C4, c1 = (w1 - j0) * C4;
      float s = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const float4 a = row0[c0 + LPR * v], bq = row0[c1 + LPR * v], c = row1[c0 + LPR * v], d = row1[c1 + LPR * v];
        x[px][v].x = (1.f - fh) * ((1.f - fw) * a.x + fw * bq.x) + fh * ((1.f - fw) * c.x + fw * d.x);
        x[px][v].y = (1.f - fh) * ((1.f - fw) * a.y + fw * bq.y) + fh * ((1.f - fw) * c.y + fw * d.y);
        x[px][v].z = (1.f - fh) * ((1.f - fw) * a.z + fw * bq.z) + fh * ((1.f - fw) * c.z + fw * d.z);
        x[px][v].w = (1.f - fh) * ((1.f - fw) * a.w + fw * bq.w) + fh * ((1.f - fw) * c.w + fw * d.w);
        s += (x[px][v].x + x[px][v].y) + (x[px][v].z + x[px][v].w);
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      mean[px] = s / (float)C;
      float q = 0.f;
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const float dx = x[px][v].x - mean[px], dy = x[px][v].y - mean[px], dz = x[px][v].z - mean[px], dw = x[px][v].w - mean[px];
        q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
      rstd[px] = rsqrtf(q / (float)C + eps);
    }
    float acc[PX][NCLS];
#pragma unroll
    for (int px = 0; px < PX; ++px)
#pragma unroll
      for (int c = 0; c < NCLS; ++c) acc[px][c] = 0.f;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      float4 o[PX];
#pragma unroll
      for (int px = 0; px < PX; ++px) {
        o[px].x = fmaf((x[px][v].x - mean[px]) * rstd[px], g[v].x, bt[v].x);
        o[px].y = fmaf((x[px][v].y - mean[px]) * rstd[px], g[v].y, bt[v].y);
        o[px].z = fmaf((x[px][v].z - mean[px]) * rstd[px], g[v].z, bt[v].z);
        o[px].w = fmaf((x[px][v].w - mean[px]) * rstd[px], g[v].w, bt[v].w);
      }
#pragma unroll
      for (int c = 0; c < NCLS; ++c) {
        const float4 wv = *reinterpret_cast<const float4 *>(&sw[c * C + 4 * (l + LPR * v)]);
#pragma unroll
        for (int px = 0; px < PX; ++px)
          acc[px][c] = fmaf(o[px].x, wv.x, fmaf(o[px].y, wv.y, fmaf(o[px].z, wv.z, fmaf(o[px].w, wv.w, acc[px][c]))));
      }
    }
#pragma unroll
    for (int px = 0; px < PX; ++px)
#pragma unroll
      for (int c = 0; c < NCLS; ++c) {
        float a = acc[px][c];
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (l == 0) mylog[c * 32 + (pass * PX + px) * RPW + sub] = a;
      }
  }
  __syncwarp();
  // this warp's 32 consecutive pixels of output row oh x NCLS classes -> NCHW: one 128-byte run per class
  const int ow = ow_t + lane;
  if (ow < Wo) {
    float *op = out + ((long long)b * NCLS * Ho + oh) * Wo + ow;
#pragma unroll
    for (int c = 0; c < NCLS; ++c) op[(long long)c * Ho * Wo] = mylog[c * 32 + lane];
  }
}

template <int NCLS>
static bool upsample2x_norm_head_fast(const float *in, const float *gamma, const float *beta, const float *wcls, float *out,
                                      int B, int Hin, int Win, int C, float eps, cudaStream_t stream) {
  if (NCLS == 0 || NCLS > 24) return false;
  const long long npix = 4LL * B * Hin * Win;
  (void)npix;
  if (B > 65535 || (2 * Hin + UH_TH - 1) / UH_TH > 65535) return false;
#define TRY(LPR, V)                                                                                                         \
  if (C == 4 * (LPR) * (V)) {                                                                                               \
    constexpr int NC = (NCLS > 0 && NCLS <= 24 ? NCLS : 1);                                                                 \
    auto kern = upsample2x_norm_head_fast_kernel<LPR, V, NC>;                                                               \
    const size_t smem = sizeof(float) * ((size_t)UH_IH * UH_IW * C + (size_t)NC * C + 8 * NC * 32);                         \
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return false;    \
    dim3 grid((2 * Win + UH_TW - 1) / UH_TW, (2 * Hin + UH_TH - 1) / UH_TH, B);                                             \
    kern<<<grid, 256, smem, stream>>>(in, gamma, beta, wcls, out, B, Hin, Win, eps);                                        \
    return true;                                                                                                            \
  }
  TRY(8, 2) TRY(8, 3) TRY(8, 4) TRY(16, 3) TRY(16, 4)
#undef TRY
  return false;
}

template <int NCLS>
static int upsample2x_norm_dispatch(const float *in, const float *gamma, const float *beta, const float *wcls, float *out,
                                    int B, int Hin, int Win, int C, float eps, cudaStream_t stream) {
  const long long npix = 4LL * B * Hin * Win;
  if (NCLS == 0 && gamma == nullptr) {   // plain bilinear x2
    const long long per_img = 4LL * Hin * Win * (C >> 2);
    if (per_img >= (1LL << 31)) { set_error("upsample2x: image too large for 32-bit indexing"); return SIGMA_EUNSUPPORTED; }
    dim3 grid((unsigned)std::min<long long>((per_img + 255) / 256, kNumSMs * 8), (unsigned)B);
    upsample2x_plain_kernel<<<grid, 256, 0, stream>>>(in, out, B, Hin, Win, C);
    SIGMA_CHECK_LAUNCH();
    return SIGMA_OK;
  }
  if (NCLS > 0 && upsample2x_norm_head_fast<NCLS>(in, gamma, beta, wcls, out, B, Hin, Win, C, eps, stream)) {
    SIGMA_CHECK_LAUNCH();
    return SIGMA_OK;
  }
  const int ppc = NCLS > 0 ? 32 : 8;
  const unsigned grid = (unsigned)((npix + ppc - 1) / ppc);
  const int nvec = C >> 2;
#define LAUNCH(MV) upsample2x_norm_kernel<MV, NCLS><<<grid, 256, 0, stream>>>(in, gamma, beta, wcls, out, B, Hin, Win, C, eps)
  if (nvec <= 32) LAUNCH(1);
  else if (nvec <= 64) LAUNCH(2);
  else if (nvec <= 128) LAUNCH(4);
  else if (nvec <= 256) LAUNCH(8);
  else { set_error("upsample2x_norm: C=%d > 1024 unsupported", C); return SIGMA_EUNSUPPORTED; }
#undef LAUNCH
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

int upsample2x_norm_launch(const float *in, const float *gamma, const float *beta, const float *wcls, int ncls, float *out,
                           int B, int Hin, int Win, int C, float eps, cudaStream_t stream) {
  switch (ncls) {
    case 0: return upsample2x_norm_dispatch<0>(in, gamma, beta, wcls, out, B, Hin, Win, C, eps, stream);
#define CASE(n) case n: return upsample2x_norm_dispatch<n>(in, gamma, beta, wcls, out, B, Hin, Win, C, eps, stream);
    CASE(2) CASE(3) CASE(4) CASE(5) CASE(6) CASE(7) CASE(8) CASE(9) CASE(10) CASE(11) CASE(12) CASE(13) CASE(14) CASE(16)
    CASE(19) CASE(20) CASE(21) CASE(37) CASE(40) CASE(41)
#undef CASE
  }
  set_error("upsample2x_norm: num_classes=%d has no fused head instantiation", ncls);
  return SIGMA_EUNSUPPORTED;
}

// ---- channel attention pooling: per (image, channel) mean and max over H·W, channels-last ----
// partial[b][s][0][c] = sum, partial[b][s][1][c] = max over the s-th slice of positions
__global__ void __launch_bounds__(256) pool_avgmax_partial_kernel(const float *__restrict__ x, float *__restrict__ partial,
                                                                 long long L, int C, int nslice) {
  extern __shared__ float sred[];  // [2][rows][C]
  const int b = blockIdx.y, s = blockIdx.x;
  const int nvec = C >> 2;
  const int rows = blockDim.x / nvec;          // position rows processed per iteration
  const int cq = threadIdx.x % nvec, pr = threadIdx.x / nvec;
  const long long per = (L + nslice - 1) / nslice;
  const long long l0 = (long long)s * per, l1 = min(L, l0 + per);
  float4 sm = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 mx = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  if (pr < rows) {
    const float4 *xb = reinterpret_cast<const float4 *>(x + (long long)b * L * C) + cq;
    for (long long l = l0 + pr; l < l1; l += rows) {
      const float4 v = __ldg(xb + l * nvec);
      sm.x += v.x; sm.y += v.y; sm.z += v.z; sm.w += v.w;
      mx.x = fmaxf(mx.x, v.x); mx.y = fmaxf(mx.y, v.y); mx.z = fmaxf(mx.z, v.z); mx.w = fmaxf(mx.w, v.w);
    }
    float *ps = sred + (size_t)pr * C + 4 * cq;
    float *pm = sred + (size_t)rows * C + (size_t)pr * C + 4 * cq;
    ps[0] = sm.x; ps[1] = sm.y; ps[2] = sm.z; ps[3] = sm.w;
    pm[0] = mx.x; pm[1] = mx.y; pm[2] = mx.z; pm[3] = mx.w;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float a = 0.f, m = -INFINITY;
    for (int r = 0; r < rows; ++r) {
      a += sred[(size_t)r * C + c];
      m = fmaxf(m, sred[(size_t)rows * C + (size_t)r * C + c]);
    }
    float *o = partial + (((long long)b * nslice + s) * 2) * C;
    o[c] = a;
    o[C + c] = m;
  }
}

int pool_avgmax_partial_launch(const float *x, float *partial, int B, long long L, int C, int nslice, cudaStream_t stream) {
  const int nvec = C >> 2;
  if (nvec > 256) { set_error("pool_avgmax: C=%d > 1024 unsupported", C); return SIGMA_EUNSUPPORTED; }
  const int rows = 256 / nvec;
  const size_t smem = 2 * (size_t)rows * C * sizeof(float);
  dim3 grid(nslice, B);
  pool_avgmax_partial_kernel<<<grid, 256, smem, stream>>>(x, partial, L, C, nslice);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

// out[r,:] = a[r,:]·sa[b(r),:] + b[r,:]·sb[:]      (CVSSDecoderBlock tail: CAB·sigmoid(attn) + x·scale2, vmamba.py:1741,1803;
// with a = NULL: out = b·sb, the x·scale1 residual of vmamba.py:1801)
__global__ void __launch_bounds__(256) scale_add_kernel(const float4 *__restrict__ a, const float *__restrict__ sa,
                                                       const float4 *__restrict__ bq, const float *__restrict__ sb,
                                                       float4 *__restrict__ out, long long nvec_total, int nvec,
                                                       long long rows_per_batch) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec_total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / nvec;
    const int c = (int)(i - r * nvec);
    const float4 vb = __ldg(bq + i);
    const float4 s2 = __ldg(reinterpret_cast<const float4 *>(sb) + c);
    float4 o = make_float4(vb.x * s2.x, vb.y * s2.y, vb.z * s2.z, vb.w * s2.w);
    if (a != nullptr) {
      const float4 va = __ldg(a + i);
      const float4 s1 = __ldg(reinterpret_cast<const float4 *>(sa) + (r / rows_per_batch) * nvec + c);
      o.x = fmaf(va.x, s1.x, o.x); o.y = fmaf(va.y, s1.y, o.y); o.z = fmaf(va.z, s1.z, o.z); o.w = fmaf(va.w, s1.w, o.w);
    }
    out[i] = o;
  }
}

int scale_add_launch(const float *a, const float *sa, const float *b, const float *sb, float *out, long long rows,
                     long long rows_per_batch, int C, cudaStream_t stream) {
  const long long tot = rows * (C >> 2);
  if (tot == 0) return SIGMA_OK;
  const unsigned grid = (unsigned)std::min<long long>((tot + 255) / 256, kNumSMs * 32);
  scale_add_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const float4 *>(a), sa, reinterpret_cast<const float4 *>(b), sb,
                                             reinterpret_cast<float4 *>(out), tot, C >> 2, rows_per_batch);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

}  // namespace sigma
