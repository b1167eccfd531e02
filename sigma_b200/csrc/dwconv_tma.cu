// Depthwise 3x3 (pad 1) + bias + SiLU on channels-last fp32 (vmamba.py:683-692,1072), TMA-tiled.
//
// A CTA owns a block of 32 channels (128 bytes of every pixel row) and walks spatial tiles of 8 x 16 output pixels
// persistently.  Each tile's (8+2) x (16+2) x 32-channel input halo is ONE TMA box: out-of-bounds coordinates
// (-1, H, W, channels >= D) are zero-filled by the TMA unit, which is exactly the convolution's zero padding, and
// the x operand may be a strided view (the x half of in_proj's [x | z] rows).  DC_NSLOT ring slots: the boxes of the
// next DC_NSLOT-1 tiles are in flight while the current one is computed (a tile's compute is ~1/3 of its HBM time, so
// with 2 slots the CTAs mostly waited for the one box in flight: 65 % of the HBM roofline).  A thread produces 2 rows x 4 columns x 4 channels from a 4 x 6
// window read from shared memory (24 LDS.128 for 8 float4 outputs); the 9 taps of its channels live in registers.
// HBM-bound: 8 bytes per output element (4 read + 4 written; halo re-reads hit L2).
// The first version of this kernel read its window straight from global memory through L1 (18 loads per 4
// outputs, no prefetch across loop iterations) and reached ~35 % of the HBM roofline.
#include <algorithm>
#include <type_traits>
#include "common.cuh"
#include "tma.cuh"

namespace sigma {

constexpr int DC_CB = 32, DC_TW = 16, DC_TH = 8, DC_NSLOT = 4;
constexpr int DC_THREADS = 8 * (DC_TW / 4) * (DC_TH / 2);          // 8 channel quads x column groups x row pairs
constexpr int DC_TILE_FL = DC_CB * (DC_TW + 2) * (DC_TH + 2);

struct DwTmaParams {
  CUtensorMap map;
  const float *w, *bias;
  void *y;
  long long y_batch_stride;
  int batch, H, W, D, tiles_w, tiles_h;
  long long ntiles;
};

// T: element type of x and y (float, or __nv_bfloat16 / __half in the bf16 / fp16 inference modes: same tiles at half the bytes;
// weights, bias and the accumulation stay fp32)
template <typename T>
__global__ void __launch_bounds__(DC_THREADS, 2) dwconv3x3_silu_tma_kernel(const __grid_constant__ DwTmaParams p) {
  constexpr int DC_TILE_BYTES = DC_TILE_FL * (int)sizeof(T);
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  T *tiles = reinterpret_cast<T *>(smem_raw);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + DC_NSLOT * DC_TILE_BYTES);
  __shared__ __align__(16) float sw[9][DC_CB];
  __shared__ __align__(16) float sb[DC_CB];

  const int tid = threadIdx.x;
  const int c0 = blockIdx.x * DC_CB;
  for (int i = tid; i < 9 * DC_CB; i += blockDim.x) {
    const int c = i / 9, tap = i - c * 9;
    sw[tap][c] = (c0 + c < p.D) ? p.w[(long long)(c0 + c) * 9 + tap] : 0.f;
  }
  for (int i = tid; i < DC_CB; i += blockDim.x) sb[i] = (p.bias && c0 + i < p.D) ? p.bias[c0 + i] : 0.f;
  if (tid == 0) {
    for (int i = 0; i < DC_NSLOT; ++i) mbar_init(&full[i], 1);
    fence_mbar_init();
    tma_prefetch_desc(&p.map);
  }
  __syncthreads();

  const int cq = tid & 7, wg = (tid >> 3) % (DC_TW / 4), hp = (tid >> 3) / (DC_TW / 4);   // channel quad, column group, row pair
  float4 wt[9];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) wt[tap] = *reinterpret_cast<const float4 *>(&sw[tap][4 * cq]);
  const float4 bv = *reinterpret_cast<const float4 *>(&sb[4 * cq]);
  const int c = c0 + 4 * cq;
  const long long tiles_per_img = (long long)p.tiles_w * p.tiles_h;

  auto issue = [&](long long t, int st) {
    const int b = (int)(t / tiles_per_img);
    const int r = (int)(t - (long long)b * tiles_per_img);
    const int th = r / p.tiles_w, tw = r - th * p.tiles_w;
    mbar_arrive_expect_tx(&full[st], DC_TILE_BYTES);
    tma_load_4d(tiles + st * DC_TILE_FL, &p.map, &full[st], c0, tw * DC_TW - 1, th * DC_TH - 1, b);
  };

  long long t = blockIdx.y;
  if (tid == 0)
    for (int k = 0; k < DC_NSLOT - 1; ++k)
      if (t + (long long)k * gridDim.y < p.ntiles) issue(t + (long long)k * gridDim.y, k);
  int st = 0, ph = 0;
  for (int it = 0; t < p.ntiles; t += gridDim.y, ++it) {
    const long long tn = t + (long long)(DC_NSLOT - 1) * gridDim.y;
    // the slot of tile it-1 was released by the barrier that ended iteration it-1: refill it with tile it+NSLOT-1
    if (tid == 0 && tn < p.ntiles) issue(tn, st == 0 ? DC_NSLOT - 1 : st - 1);
    mbar_wait(&full[st], (uint32_t)ph);

    const int b = (int)(t / tiles_per_img);
    const int r = (int)(t - (long long)b * tiles_per_img);
    const int th = r / p.tiles_w, tw = r - th * p.tiles_w;
    const T *base = tiles + st * DC_TILE_FL + ((2 * hp) * (DC_TW + 2) + 4 * wg) * DC_CB + 4 * cq;
    float4 acc[2][4];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[rr][j] = bv;
#pragma unroll
    for (int wr = 0; wr < 4; ++wr) {       // window row wr feeds output row 0 with tap row wr and output row 1 with tap row wr-1
      float4 win[6];
#pragma unroll
      for (int j = 0; j < 6; ++j) win[j] = ld4(base + (wr * (DC_TW + 2) + j) * DC_CB);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int tr = wr - rr;
        if (tr < 0 || tr > 2) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
          for (int dx = 0; dx < 3; ++dx) {
            const float4 v = win[j + dx];
            const float4 k = wt[tr * 3 + dx];
            // four FMAs as two pairs (common.cuh: fma2)
            const f2 lo = fma2(f2{v.x, v.y}, f2{k.x, k.y}, f2{acc[rr][j].x, acc[rr][j].y});
            const f2 hi = fma2(f2{v.z, v.w}, f2{k.z, k.w}, f2{acc[rr][j].z, acc[rr][j].w});
            acc[rr][j] = make_float4(lo.x, lo.y, hi.x, hi.y);
          }
        }
      }
    }
    if (c < p.D) {
      const int h0 = th * DC_TH + 2 * hp, w0 = tw * DC_TW + 4 * wg;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int h = h0 + rr;
        if (h >= p.H) continue;
        T *yb = reinterpret_cast<T *>(p.y) + (long long)b * p.y_batch_stride + ((long long)h * p.W + w0) * p.D + c;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (w0 + j < p.W) {
            float4 o;
            o.x = silu(acc[rr][j].x); o.y = silu(acc[rr][j].y); o.z = silu(acc[rr][j].z); o.w = silu(acc[rr][j].w);
            st4(yb + (long long)j * p.D, o);
          }
        }
      }
    }
    __syncthreads();   // every thread is done reading slot st before it is refilled
    if (++st == DC_NSLOT) { st = 0; ph ^= 1; }
  }
}

template <typename T>
static int dwconv_tma_launch(const T *x, long long x_row_stride, long long x_batch_stride, const float *w, const float *bias, T *y,
                             long long y_batch_stride, int batch, int H, int W, int D, cudaStream_t stream) {
  constexpr int es = (int)sizeof(T);
  DwTmaParams p;
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)W, (uint64_t)H, (uint64_t)batch};
  const uint64_t str[3] = {(uint64_t)x_row_stride * es, (uint64_t)W * x_row_stride * es, (uint64_t)x_batch_stride * es};
  const uint32_t box[4] = {DC_CB, DC_TW + 2, DC_TH + 2, 1};
  const CUtensorMapDataType dt = es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : std::is_same<T, __half>::value ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  int rc = make_tmap(&p.map, dt, 4, x, dims, str, box, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  if (rc) return rc;
  p.w = w; p.bias = bias; p.y = y; p.y_batch_stride = y_batch_stride;
  p.batch = batch; p.H = H; p.W = W; p.D = D;
  p.tiles_w = (W + DC_TW - 1) / DC_TW;
  p.tiles_h = (H + DC_TH - 1) / DC_TH;
  p.ntiles = (long long)batch * p.tiles_w * p.tiles_h;
  if (p.ntiles == 0) return SIGMA_OK;
  const int cblocks = (D + DC_CB - 1) / DC_CB;
  const size_t smem = (size_t)DC_NSLOT * DC_TILE_FL * es + 64;
  SIGMA_CHECK_CUDA(cudaFuncSetAttribute(dwconv3x3_silu_tma_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // persistent over spatial tiles: 2 CTAs per SM in total, channel block fastest so that the CTAs working on one
  // spatial tile (adjacent 128-byte pieces of the same pixel rows) run at the same time
  const long long slots = kNumSMs * 2;
  // (never more CTAs than resident slots: a partial second wave of persistent CTAs would double the kernel time)
  const unsigned ny = (unsigned)std::max<long long>(1, std::min<long long>(p.ntiles, slots / cblocks));
  dim3 grid(cblocks, ny);
  dwconv3x3_silu_tma_kernel<T><<<grid, DC_THREADS, smem, stream>>>(p);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

int dwconv3x3_silu_fwd_launch(int dtype, const void *x, long long x_row_stride, long long x_batch_stride, const float *w,
                              const float *bias, void *y, long long y_batch_stride, int batch, int H, int W, int D, cudaStream_t stream) {
  if (dtype == SIGMA_F32)
    return dwconv_tma_launch<float>((const float *)x, x_row_stride, x_batch_stride, w, bias, (float *)y, y_batch_stride, batch, H, W,
                                    D, stream);
  if (dtype == SIGMA_F16)
    return dwconv_tma_launch<__half>((const __half *)x, x_row_stride, x_batch_stride, w, bias, (__half *)y, y_batch_stride, batch, H,
                                     W, D, stream);
  return dwconv_tma_launch<__nv_bfloat16>((const __nv_bfloat16 *)x, x_row_stride, x_batch_stride, w, bias, (__nv_bfloat16 *)y,
                                          y_batch_stride, batch, H, W, D, stream);
}

// ---- backward (training): y = SiLU(pre), pre = conv3x3(x) + b; dy -> dx, dw, db ----
// The pre-activation is recomputed from x, so the forward saves nothing but x.  Per 8 x 16 output tile and 32-channel block, two
// TMA boxes land in one ring slot: x with a 2-pixel halo (12 x 20) and dy with a 1-pixel halo (10 x 18).  Zero fill gives the
// padding, and dy = 0 outside the image makes g = 0 there.  Then:
//   phase 1: g = dy·s·(1 + pre·(1 − s)), s = sigmoid(pre), on the 10 x 18 one-halo region, fp32 in shared memory (in place of the dy
//            box for fp32, whose size it has; a separate buffer for 16-bit dy);
//   phase 2: dx = the transposed (flipped) stencil of g on the tile; dw[c, tap] += g·(x at the tap's shift) and db += g over the
//            tile's own pixels, in registers.
// x and dy are read once and dx written once (12 B per element in fp32, 6 B in 16-bit; halo re-reads hit L2).  Deterministic by
// construction: each persistent CTA walks its tiles in a fixed order, sums its threads' dw / db in a fixed order into one partial
// row of the workspace, and sum_parts_det_kernel adds the rows in order.  No float atomics.
constexpr int DB_NSLOT = 2;                                     // two slots keep two CTAs per SM in fp32 (105 KB of ring each)
constexpr int DB_XW = DC_TW + 4, DB_GW = DC_TW + 2;             // x box / g region widths
constexpr int DB_XTILE = DC_CB * DB_XW * (DC_TH + 4);
constexpr int DB_GTILE = DC_CB * DB_GW * (DC_TH + 2);           // = DC_TILE_FL
constexpr int DB_UNITS = DC_THREADS / 8;                        // 16 pixel units per channel quad

struct DwBwdParams {
  CUtensorMap xmap, dymap;
  const float *w, *bias;
  void *dx;
  float *part_w, *part_b;                                       // (gridDim.y, 9·D) and (gridDim.y, D) partial rows
  long long dx_batch_stride;
  int H, W, D, tiles_w, tiles_h;
  long long ntiles;
};

__device__ __forceinline__ void fma4(float4 &a, float4 v, float4 k) {
  const f2 lo = fma2(f2{v.x, v.y}, f2{k.x, k.y}, f2{a.x, a.y});
  const f2 hi = fma2(f2{v.z, v.w}, f2{k.z, k.w}, f2{a.z, a.w});
  a = make_float4(lo.x, lo.y, hi.x, hi.y);
}

__device__ __forceinline__ float silu_grad(float pre, float d) {
  const float s = __fdividef(1.f, 1.f + ex2(-pre * kLog2e));
  return d * s * fmaf(pre, 1.f - s, 1.f);
}

template <typename T>
__global__ void __launch_bounds__(DC_THREADS, 2) dwconv3x3_silu_bwd_tma_kernel(const __grid_constant__ DwBwdParams p) {
  constexpr bool kGInPlace = sizeof(T) == sizeof(float);
  constexpr int XB = DB_XTILE * (int)sizeof(T), SLOT = XB + DB_GTILE * (int)sizeof(T);
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  float *gsep = reinterpret_cast<float *>(smem_raw + DB_NSLOT * SLOT);
  uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + DB_NSLOT * SLOT + (kGInPlace ? 0 : DB_GTILE * 4));
  __shared__ __align__(16) float sw[9][DC_CB];
  __shared__ __align__(16) float sb[DC_CB];

  const int tid = threadIdx.x;
  const int c0 = blockIdx.x * DC_CB;
  for (int i = tid; i < 9 * DC_CB; i += blockDim.x) {
    const int c = i / 9, tap = i - c * 9;
    sw[tap][c] = (c0 + c < p.D) ? p.w[(long long)(c0 + c) * 9 + tap] : 0.f;
  }
  for (int i = tid; i < DC_CB; i += blockDim.x) sb[i] = (p.bias && c0 + i < p.D) ? p.bias[c0 + i] : 0.f;
  if (tid == 0) {
    for (int i = 0; i < DB_NSLOT; ++i) mbar_init(&full[i], 1);
    fence_mbar_init();
    tma_prefetch_desc(&p.xmap);
    tma_prefetch_desc(&p.dymap);
  }
  __syncthreads();

  const int cq = tid & 7, unit = tid >> 3;
  const int wg = unit % (DC_TW / 4), hp = unit / (DC_TW / 4);   // phase 2: column group (4 pixels), row pair of the tile
  const int gv = unit % 3, gu = unit / 3;                         // phase 1: column sextet, row pair of the g region (unit 15 idles)
  float4 wt[9];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) wt[tap] = *reinterpret_cast<const float4 *>(&sw[tap][4 * cq]);
  const float4 bv = *reinterpret_cast<const float4 *>(&sb[4 * cq]);
  const int c = c0 + 4 * cq;
  const long long tiles_per_img = (long long)p.tiles_w * p.tiles_h;
  float4 dwa[9], dba = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int k = 0; k < 9; ++k) dwa[k] = dba;

  auto issue = [&](long long t, int st) {
    const int b = (int)(t / tiles_per_img);
    const int r = (int)(t - (long long)b * tiles_per_img);
    const int th = r / p.tiles_w, tw = r - th * p.tiles_w;
    unsigned char *slot = smem_raw + st * SLOT;
    mbar_arrive_expect_tx(&full[st], SLOT);
    tma_load_4d(slot, &p.xmap, &full[st], c0, tw * DC_TW - 2, th * DC_TH - 2, b);
    tma_load_4d(slot + XB, &p.dymap, &full[st], c0, tw * DC_TW - 1, th * DC_TH - 1, b);
  };

  long long t = blockIdx.y;
  if (tid == 0)
    for (int k = 0; k < DB_NSLOT - 1; ++k)
      if (t + (long long)k * gridDim.y < p.ntiles) issue(t + (long long)k * gridDim.y, k);
  int st = 0, ph = 0;
  for (; t < p.ntiles; t += gridDim.y) {
    const long long tn = t + (long long)(DB_NSLOT - 1) * gridDim.y;
    // the slot of the previous tile was released by the barrier that ended its iteration
    if (tid == 0 && tn < p.ntiles) issue(tn, st == 0 ? DB_NSLOT - 1 : st - 1);
    mbar_wait(&full[st], (uint32_t)ph);

    const T *xs = reinterpret_cast<const T *>(smem_raw + st * SLOT);
    const T *dys = reinterpret_cast<const T *>(smem_raw + st * SLOT + XB);
    float *g = kGInPlace ? reinterpret_cast<float *>(smem_raw + st * SLOT + XB) : gsep;

    // phase 1: 2 rows x 6 columns of g per thread from a 4 x 8 window of x (each g element is read as dy and written as g by the
    // same thread, so the in-place fp32 buffer has no hazard)
    if (gu < (DC_TH + 2) / 2) {
      float4 acc[2][6];
#pragma unroll
      for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int j = 0; j < 6; ++j) acc[rr][j] = bv;
      const T *xb = xs + ((2 * gu) * DB_XW + 6 * gv) * DC_CB + 4 * cq;
#pragma unroll
      for (int xr = 0; xr < 4; ++xr) {
        float4 win[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) win[j] = ld4(xb + (xr * DB_XW + j) * DC_CB);
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int tr = xr - rr;
          if (tr < 0 || tr > 2) continue;
#pragma unroll
          for (int j = 0; j < 6; ++j)
#pragma unroll
            for (int dxx = 0; dxx < 3; ++dxx) fma4(acc[rr][j], win[j + dxx], wt[tr * 3 + dxx]);
        }
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          const int off = ((2 * gu + rr) * DB_GW + 6 * gv + j) * DC_CB + 4 * cq;
          const float4 d = ld4(dys + off), a = acc[rr][j];
          *reinterpret_cast<float4 *>(g + off) =
              make_float4(silu_grad(a.x, d.x), silu_grad(a.y, d.y), silu_grad(a.z, d.z), silu_grad(a.w, d.w));
        }
      if (kGInPlace) fence_proxy_async();   // g overwrote the dy box by the generic proxy: order it before the slot's next TMA write
    }
    __syncthreads();

    // phase 2: dx of 2 rows x 4 columns from a 4 x 6 window of g (flipped taps), keeping g of the thread's own pixels ...
    const int b = (int)(t / tiles_per_img);
    const int r = (int)(t - (long long)b * tiles_per_img);
    const int th = r / p.tiles_w, tw = r - th * p.tiles_w;
    float4 own[2][4], acc[2][4];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[rr][j] = make_float4(0.f, 0.f, 0.f, 0.f);
    const float *gb = g + ((2 * hp) * DB_GW + 4 * wg) * DC_CB + 4 * cq;
#pragma unroll
    for (int wr = 0; wr < 4; ++wr) {       // g row wr feeds output row rr with tap row 2 - (wr - rr)
      float4 win[6];
#pragma unroll
      for (int j = 0; j < 6; ++j) win[j] = *reinterpret_cast<const float4 *>(gb + (wr * DB_GW + j) * DC_CB);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        if (wr == rr + 1)
#pragma unroll
          for (int j = 0; j < 4; ++j) own[rr][j] = win[j + 1];
        const int rel = wr - rr;
        if (rel < 0 || rel > 2) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int dxx = 0; dxx < 3; ++dxx) fma4(acc[rr][j], win[j + dxx], wt[(2 - rel) * 3 + 2 - dxx]);
      }
    }
    if (c < p.D) {
      const int h0 = th * DC_TH + 2 * hp, w0 = tw * DC_TW + 4 * wg;
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int h = h0 + rr;
        if (h >= p.H) continue;
        T *dxb = reinterpret_cast<T *>(p.dx) + (long long)b * p.dx_batch_stride + ((long long)h * p.W + w0) * p.D + c;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (w0 + j < p.W) st4(dxb + (long long)j * p.D, acc[rr][j]);
      }
    }
    // ... and dw / db of those pixels from a 4 x 6 window of x (x box row 2·hp + 1 + xr is tap row xr - rr of output row rr)
    const T *xb = xs + ((2 * hp + 1) * DB_XW + 4 * wg + 1) * DC_CB + 4 * cq;
#pragma unroll
    for (int xr = 0; xr < 4; ++xr) {
      float4 win[6];
#pragma unroll
      for (int j = 0; j < 6; ++j) win[j] = ld4(xb + (xr * DB_XW + j) * DC_CB);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int tr = xr - rr;
        if (tr < 0 || tr > 2) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int dxx = 0; dxx < 3; ++dxx) fma4(dwa[tr * 3 + dxx], own[rr][j], win[j + dxx]);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr)
#pragma unroll
      for (int j = 0; j < 4; ++j) dba = make_float4(dba.x + own[rr][j].x, dba.y + own[rr][j].y, dba.z + own[rr][j].z, dba.w + own[rr][j].w);
    __syncthreads();   // every thread is done with slot st (and g) before either is written again
    if (++st == DB_NSLOT) { st = 0; ph ^= 1; }
  }

  // the CTA's partial row: the 16 units' sums of each channel added in unit order, in the idle ring (every box issued was waited for)
  float *red = reinterpret_cast<float *>(smem_raw);             // [unit][10][DC_CB]: taps 0..8, then db
#pragma unroll
  for (int k = 0; k < 9; ++k) *reinterpret_cast<float4 *>(&red[(unit * 10 + k) * DC_CB + 4 * cq]) = dwa[k];
  *reinterpret_cast<float4 *>(&red[(unit * 10 + 9) * DC_CB + 4 * cq]) = dba;
  __syncthreads();
  for (int i = tid; i < 10 * DC_CB; i += blockDim.x) {
    const int k = i / DC_CB, cc = i - k * DC_CB, ch = c0 + cc;
    float s = 0.f;
    for (int u = 0; u < DB_UNITS; ++u) s += red[(u * 10 + k) * DC_CB + cc];
    if (ch < p.D) {
      if (k < 9) p.part_w[(long long)blockIdx.y * 9 * p.D + (long long)ch * 9 + k] = s;
      else if (p.part_b) p.part_b[(long long)blockIdx.y * p.D + ch] = s;
    }
  }
}

// the launch plan of the backward: persistent CTAs per channel block (gridDim.y), which is also the number of partial rows.  A
// function of the shape alone, so the order of every sum is too.
static int dwconv_bwd_parts(int batch, int H, int W, int D) {
  const long long ntiles = (long long)batch * ((W + DC_TW - 1) / DC_TW) * ((H + DC_TH - 1) / DC_TH);
  const int cblocks = (D + DC_CB - 1) / DC_CB;
  return (int)std::max<long long>(1, std::min<long long>(ntiles, (long long)kNumSMs * 2 / cblocks));
}

size_t dwconv3x3_silu_bwd_workspace_bytes(int batch, int H, int W, int D) {
  const size_t ny = (size_t)dwconv_bwd_parts(batch, H, W, D);
  return align256(ny * 9 * D * sizeof(float)) + align256(ny * D * sizeof(float));
}

template <typename T>
static int dwconv_bwd_tma_launch(const T *x, long long x_row_stride, long long x_batch_stride, const float *w, const float *bias,
                                 const T *dy, long long dy_batch_stride, T *dx, long long dx_batch_stride, float *dw, float *db,
                                 int batch, int H, int W, int D, void *ws, cudaStream_t stream) {
  constexpr int es = (int)sizeof(T);
  const CUtensorMapDataType dt = es == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                 : std::is_same<T, __half>::value ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  // a runtime call before the tensor maps are encoded: it binds the device's context to the calling thread, which autograd's worker
  // thread (a backward that starts at this node) does not have yet, and cuTensorMapEncodeTiled would fail there
  const size_t smem = (size_t)DB_NSLOT * (DB_XTILE + DB_GTILE) * es + (es == 4 ? 0 : DB_GTILE * sizeof(float)) + 64;
  SIGMA_CHECK_CUDA(cudaFuncSetAttribute(dwconv3x3_silu_bwd_tma_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  DwBwdParams p;
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)W, (uint64_t)H, (uint64_t)batch};
  const uint64_t xstr[3] = {(uint64_t)x_row_stride * es, (uint64_t)W * x_row_stride * es, (uint64_t)x_batch_stride * es};
  const uint32_t xbox[4] = {DC_CB, DB_XW, DC_TH + 4, 1};
  int rc = make_tmap(&p.xmap, dt, 4, x, dims, xstr, xbox, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
  if (rc) return rc;
  const uint64_t ystr[3] = {(uint64_t)D * es, (uint64_t)W * D * es, (uint64_t)dy_batch_stride * es};
  const uint32_t ybox[4] = {DC_CB, DB_GW, DC_TH + 2, 1};
  if ((rc = make_tmap(&p.dymap, dt, 4, dy, dims, ystr, ybox, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))) return rc;
  const int ny = dwconv_bwd_parts(batch, H, W, D);
  p.w = w; p.bias = bias; p.dx = dx; p.dx_batch_stride = dx_batch_stride;
  p.part_w = (float *)ws;
  p.part_b = bias ? (float *)((char *)ws + align256((size_t)ny * 9 * D * sizeof(float))) : nullptr;
  p.H = H; p.W = W; p.D = D;
  p.tiles_w = (W + DC_TW - 1) / DC_TW;
  p.tiles_h = (H + DC_TH - 1) / DC_TH;
  p.ntiles = (long long)batch * p.tiles_w * p.tiles_h;
  dwconv3x3_silu_bwd_tma_kernel<T><<<dim3((D + DC_CB - 1) / DC_CB, ny), DC_THREADS, smem, stream>>>(p);
  SIGMA_CHECK_LAUNCH();
  if ((rc = sum_parts_det_launch(p.part_w, ny, 9LL * D, 9LL * D, 0, dw, stream))) return rc;
  return bias ? sum_parts_det_launch(p.part_b, ny, D, D, 0, db, stream) : SIGMA_OK;
}

int dwconv3x3_silu_bwd_launch(int dtype, const void *x, long long x_row_stride, long long x_batch_stride, const float *w,
                              const float *bias, const void *dy, long long dy_batch_stride, void *dx, long long dx_batch_stride, float *dw,
                              float *db, int batch, int H, int W, int D, void *ws, cudaStream_t stream) {
  if (dtype == SIGMA_F32)
    return dwconv_bwd_tma_launch<float>((const float *)x, x_row_stride, x_batch_stride, w, bias, (const float *)dy, dy_batch_stride,
                                        (float *)dx, dx_batch_stride, dw, db, batch, H, W, D, ws, stream);
  if (dtype == SIGMA_F16)
    return dwconv_bwd_tma_launch<__half>((const __half *)x, x_row_stride, x_batch_stride, w, bias, (const __half *)dy, dy_batch_stride,
                                         (__half *)dx, dx_batch_stride, dw, db, batch, H, W, D, ws, stream);
  return dwconv_bwd_tma_launch<__nv_bfloat16>((const __nv_bfloat16 *)x, x_row_stride, x_batch_stride, w, bias,
                                              (const __nv_bfloat16 *)dy, dy_batch_stride, (__nv_bfloat16 *)dx, dx_batch_stride, dw, db,
                                              batch, H, W, D, ws, stream);
}

}  // namespace sigma
