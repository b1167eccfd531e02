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

// returns SIGMA_OK, an error, or 1 when the shape cannot use the TMA path (caller falls back to the direct kernel)
int dwconv3x3_silu_tma_launch(const float *x, long long x_row_stride, long long x_batch_stride, const float *w,
                              const float *bias, float *y, long long y_batch_stride, int batch, int H, int W, int D,
                              cudaStream_t stream) {
  if ((x_row_stride & 3) || (x_batch_stride & 3) || ((uintptr_t)x & 15) || (D & 3)) return 1;
  return dwconv_tma_launch<float>(x, x_row_stride, x_batch_stride, w, bias, y, y_batch_stride, batch, H, W, D, stream);
}

// 16-bit x and y, dtype SIGMA_BF16 or SIGMA_F16 (the caller checks the 16-byte stride / alignment TMA needs: there is no direct
// 16-bit kernel to fall back to)
int dwconv3x3_silu_16bit_launch(int dtype, const void *x, long long x_row_stride, long long x_batch_stride, const float *w,
                                const float *bias, void *y, long long y_batch_stride, int batch, int H, int W, int D, cudaStream_t stream) {
  if (dtype == SIGMA_F16)
    return dwconv_tma_launch<__half>((const __half *)x, x_row_stride, x_batch_stride, w, bias, (__half *)y, y_batch_stride, batch, H,
                                     W, D, stream);
  return dwconv_tma_launch<__nv_bfloat16>((const __nv_bfloat16 *)x, x_row_stride, x_batch_stride, w, bias, (__nv_bfloat16 *)y,
                                          y_batch_stride, batch, H, W, D, stream);
}

}  // namespace sigma
