// Weight gradient of the dense 3x3 convolution (pad 1, stride 1) on channels-last fp32 tensors, the ChannelAttentionBlock's two
// convs in training (ops.CabConvFn):
//
//     dW[co, ci, tap] = Σ_p dy[p, co] · x[p + s(tap), ci],   db[co] = Σ_p dy[p, co],   s(tap) = (tap / 3 − 1, tap % 3 − 1)
//
// a GEMM whose K dimension is the pixels (B·H·W, up to ~10^5) and whose output (9·Cout·Cin) is small.  Both operands are
// pixel-major in channels-last memory, and wgmma reads TF32 operands from shared memory only K-major, so neither could be fed
// from a TMA box as it stands.  This kernel uses the warp-level `mma.sync.m16n8k8` TF32 MMA instead, whose fragments are
// gathered from shared memory by plain 32-bit loads in any layout: per 8 x 16 pixel patch, a CTA stages the x box with a
// one-pixel halo (10 x 18 pixels x 32 input channels; zero fill outside the image is the padding) and the dy patch (128 pixels x
// CO output channels) as they lie in memory, rows padded to 8 mod 32 words so that every fragment load is conflict-free.  Warp w
// owns tap w (9 warps): its A fragments (rows = ci, k = pixels) are read from the x box at the tap's shift — an address offset —
// and its B fragments (k = pixels, columns = co) from the dy patch, which all nine warps share.  Precision follows the forward:
// x3 = 0 issues one TF32 MMA per k-step (the hardware truncates the fp32 operands), x3 = 1 splits both operands into hi / lo in
// registers and issues A_lo·B_hi, A_hi·B_lo, A_hi·B_hi (the tf32x3 GEMM's order, small terms first).  gelu_x = 1: x is the
// pre-activation of an exact GELU, applied once per staged element (the second CAB conv reads its input's pre-activation, so the
// forward keeps no GELU output).
//
// Split-K over pixel ranges, deterministic by construction: CTA (tile, s) sums the patches of range s in order into registers
// and writes one partial row of the workspace; sum_parts_det_kernel adds the rows in order.  No float atomic.  The plan is a
// function of the shape and kNumSMs alone, so the same inputs give the same bits with or without a deterministic mode.
#include <algorithm>

#include "common.cuh"
#include "tma.cuh"

namespace sigma {

constexpr int WG_TH = 8, WG_TW = 16;                  // pixel patch (the forward conv's M tile)
constexpr int WG_PIX = WG_TH * WG_TW;                 // 128 pixels = 16 k8 steps
constexpr int WG_XH = WG_TH + 2, WG_XW = WG_TW + 2;   // x box with a one-pixel halo
constexpr int WG_CI = 32;                             // input channels per tile: two m16 fragments
constexpr int WG_XLD = WG_CI + 8;                     // x box row stride in words (≡ 8 mod 32)
constexpr int WG_THREADS = 9 * 32;                    // warp w = tap w

template <int CO> struct WgradTile {
  static constexpr int dy_ld = CO + 8;                                // ≡ 8 mod 32
  static constexpr int x_floats = WG_XH * WG_XW * WG_XLD;
  static constexpr int buf_floats = x_floats + WG_PIX * dy_ld;
  static constexpr size_t smem = 2 * buf_floats * sizeof(float);      // double buffer
};

struct WgradParams {
  const float *x, *dy;
  float *part_w, *part_b;   // (nsplit, Cout·Cin·9) in nn.Conv2d's (Cout, Cin, 3, 3) order; (nsplit, Cout), or nullptr
  int H, W, Cin, Cout, tiles_w, tiles_hw, co_tiles, nsplit, gelu_x;
  long long npatch;
};

// D[16 x 8] += A[16 x 8] · B[8 x 8]: a = rows g, g + 8, g, g + 8 / columns t, t, t + 4, t + 4; b = rows t, t + 4 / column g;
// d = (g, 2t), (g, 2t + 1), (g + 8, 2t), (g + 8, 2t + 1); g = lane / 4, t = lane % 4
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

__device__ __forceinline__ uint32_t tf32_hi(uint32_t v) { return v & 0xFFFFE000u; }
__device__ __forceinline__ uint32_t tf32_lo(uint32_t v) { return __float_as_uint(__uint_as_float(v) - __uint_as_float(v & 0xFFFFE000u)); }

template <int CO, bool X3>
__global__ void __launch_bounds__(WG_THREADS, 1) conv3x3_wgrad_kernel(const __grid_constant__ WgradParams p) {
  using T = WgradTile<CO>;
  constexpr int NT = CO / 8;   // n8 fragments per warp
  extern __shared__ __align__(16) float smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int tile = blockIdx.x, split = blockIdx.y;
  const int ci0 = (tile / p.co_tiles) * WG_CI, co0 = (tile % p.co_tiles) * CO;
  const long long pbeg = p.npatch * split / p.nsplit, pend = p.npatch * (split + 1) / p.nsplit;
  const bool do_db = p.part_b != nullptr && ci0 == 0;

  // stage patch `pt` into buffer `buf`: x box (10 x 18 pixels x 32 channels from ci0) and dy patch (128 pixels x CO from co0), as
  // 16-byte cp.async chunks whose source-size 0 outside the image or the channel range writes zeros
  auto issue = [&](long long pt, int buf) {
    const int b = (int)(pt / p.tiles_hw), r = (int)(pt - (long long)b * p.tiles_hw);
    const int y0 = (r / p.tiles_w) * WG_TH, x0 = (r % p.tiles_w) * WG_TW;
    float *xs = smem + buf * T::buf_floats, *dys = xs + T::x_floats;
    for (int i = tid; i < WG_XH * WG_XW * (WG_CI / 4); i += WG_THREADS) {
      const int pix = i / (WG_CI / 4), c = ci0 + 4 * (i % (WG_CI / 4));
      const int yy = y0 - 1 + pix / WG_XW, xx = x0 - 1 + pix % WG_XW;
      const bool ok = yy >= 0 && yy < p.H && xx >= 0 && xx < p.W && c < p.Cin;
      const float *src = ok ? p.x + (((long long)b * p.H + yy) * p.W + xx) * p.Cin + c : p.x;
      cp_async16(xs + pix * WG_XLD + 4 * (i % (WG_CI / 4)), src, ok ? 16 : 0);
    }
    for (int i = tid; i < WG_PIX * (CO / 4); i += WG_THREADS) {
      const int pix = i / (CO / 4), c = co0 + 4 * (i % (CO / 4));
      const int yy = y0 + pix / WG_TW, xx = x0 + pix % WG_TW;
      const bool ok = yy < p.H && xx < p.W && c < p.Cout;
      const float *src = ok ? p.dy + (((long long)b * p.H + yy) * p.W + xx) * p.Cout + c : p.dy;
      cp_async16(dys + pix * T::dy_ld + 4 * (i % (CO / 4)), src, ok ? 16 : 0);
    }
    cp_async_commit();
  };

  float acc[2][NT][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[h][n][i] = 0.f;
  float dbacc = 0.f;
  const int tdy = warp / 3, tdx = warp % 3;

  if (pbeg < pend) issue(pbeg, 0);
  int buf = 0;
  for (long long pt = pbeg; pt < pend; ++pt, buf ^= 1) {
    if (pt + 1 < pend) { issue(pt + 1, buf ^ 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    asm volatile("" ::: "memory");   // no shared-memory access moves above the wait
    float *xs = smem + buf * T::buf_floats;
    const float *dys = xs + T::x_floats;
    if (p.gelu_x) {   // the chunks this thread copied, which its own wait made visible to it; GELU(0) = 0 keeps the padding
      for (int i = tid; i < WG_XH * WG_XW * (WG_CI / 4); i += WG_THREADS) {
        float4 *q = reinterpret_cast<float4 *>(xs + (i / (WG_CI / 4)) * WG_XLD + 4 * (i % (WG_CI / 4)));
        float4 v = *q;
        v.x = 0.5f * v.x * (1.f + erff(v.x * 0.70710678118654752f));
        v.y = 0.5f * v.y * (1.f + erff(v.y * 0.70710678118654752f));
        v.z = 0.5f * v.z * (1.f + erff(v.z * 0.70710678118654752f));
        v.w = 0.5f * v.w * (1.f + erff(v.w * 0.70710678118654752f));
        *q = v;
      }
    }
    __syncthreads();

    // k8 step kk covers pixels 8kk .. 8kk + 7: patch row kk / 2, columns 8·(kk % 2) ..; x box pixel of tap (tdy, tdx) = (row + tdy,
    // column + tdx)
    const uint32_t *xw = reinterpret_cast<const uint32_t *>(xs), *dw = reinterpret_cast<const uint32_t *>(dys);
#pragma unroll 2
    for (int kk = 0; kk < WG_PIX / 8; ++kk) {
      const int xp = ((kk >> 1) + tdy) * WG_XW + 8 * (kk & 1) + tdx + t;
      uint32_t a[2][4], bf[NT][2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        a[h][0] = xw[xp * WG_XLD + 16 * h + g];
        a[h][1] = xw[xp * WG_XLD + 16 * h + g + 8];
        a[h][2] = xw[(xp + 4) * WG_XLD + 16 * h + g];
        a[h][3] = xw[(xp + 4) * WG_XLD + 16 * h + g + 8];
      }
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        bf[n][0] = dw[(8 * kk + t) * T::dy_ld + 8 * n + g];
        bf[n][1] = dw[(8 * kk + t + 4) * T::dy_ld + 8 * n + g];
      }
      if constexpr (X3) {
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 4; ++i) { ah[h][i] = tf32_hi(a[h][i]); al[h][i] = tf32_lo(a[h][i]); }
#pragma unroll
        for (int n = 0; n < NT; ++n) {
          const uint32_t bh[2] = {tf32_hi(bf[n][0]), tf32_hi(bf[n][1])}, bl[2] = {tf32_lo(bf[n][0]), tf32_lo(bf[n][1])};
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            mma_tf32(acc[h][n], al[h], bh);
            mma_tf32(acc[h][n], ah[h], bl);
            mma_tf32(acc[h][n], ah[h], bh);
          }
        }
      } else {
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
          for (int h = 0; h < 2; ++h) mma_tf32(acc[h][n], a[h], bf[n]);
      }
    }
    if (do_db && tid < CO)
      for (int q = 0; q < WG_PIX; ++q) dbacc += dys[q * T::dy_ld + tid];
    __syncthreads();   // every warp is done with this buffer before the next iteration's issue overwrites it
  }

  // the CTA's partial row: (co, ci, tap) at (co·Cin + ci)·9 + tap
  float *pw = p.part_w + (long long)split * p.Cout * p.Cin * 9;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int ci = ci0 + 16 * h + g + 8 * (i >> 1), co = co0 + 8 * n + 2 * t + (i & 1);
        if (ci < p.Cin && co < p.Cout) pw[((long long)co * p.Cin + ci) * 9 + warp] = acc[h][n][i];
      }
  if (do_db && tid < CO && co0 + tid < p.Cout) p.part_b[(long long)split * p.Cout + co0 + tid] = dbacc;
}

// output channels per tile: 64 when Cout is a multiple of 64 (Sigma's 64 / 128 / 192 / 384), else 32 (32, 96, ragged counts)
static int wgrad_co(int Cout) { return Cout % 64 == 0 ? 64 : 32; }

// out4 = {CO, output tiles, partial rows, CTAs}.  As many pixel ranges as fill the SMs in one wave (one CTA per SM, for the shared
// memory of the double buffer: a second, partial wave would double the time of the call), none of them empty.
void conv3x3_wgrad_plan(int batch, int H, int W, int Cin, int Cout, long long *out4) {
  const int co = wgrad_co(Cout);
  const long long tiles = (long long)((Cin + WG_CI - 1) / WG_CI) * ((Cout + co - 1) / co);
  const long long npatch = (long long)batch * ((H + WG_TH - 1) / WG_TH) * ((W + WG_TW - 1) / WG_TW);
  const long long nsplit = std::max(1LL, std::min(npatch, kNumSMs / tiles));
  out4[0] = co; out4[1] = tiles; out4[2] = nsplit; out4[3] = tiles * nsplit;
}

size_t conv3x3_wgrad_workspace_bytes(int batch, int H, int W, int Cin, int Cout) {
  long long pl[4];
  conv3x3_wgrad_plan(batch, H, W, Cin, Cout, pl);
  return align256((size_t)pl[2] * Cout * Cin * 9 * sizeof(float)) + align256((size_t)pl[2] * Cout * sizeof(float));
}

int conv3x3_wgrad_launch(const float *x, int gelu_x, const float *dy, float *dw, float *db, int batch, int H, int W, int Cin, int Cout,
                         int x3, void *ws, cudaStream_t stream) {
  long long pl[4];
  conv3x3_wgrad_plan(batch, H, W, Cin, Cout, pl);
  WgradParams p;
  p.x = x; p.dy = dy;
  p.part_w = (float *)ws;
  p.part_b = db ? (float *)((char *)ws + align256((size_t)pl[2] * Cout * Cin * 9 * sizeof(float))) : nullptr;
  p.H = H; p.W = W; p.Cin = Cin; p.Cout = Cout;
  p.tiles_w = (W + WG_TW - 1) / WG_TW;
  p.tiles_hw = p.tiles_w * ((H + WG_TH - 1) / WG_TH);
  p.co_tiles = (Cout + (int)pl[0] - 1) / (int)pl[0];
  p.nsplit = (int)pl[2];
  p.gelu_x = gelu_x;
  p.npatch = (long long)batch * p.tiles_hw;
  const void *kern = pl[0] == 64 ? (x3 ? (const void *)conv3x3_wgrad_kernel<64, true> : (const void *)conv3x3_wgrad_kernel<64, false>)
                                 : (x3 ? (const void *)conv3x3_wgrad_kernel<32, true> : (const void *)conv3x3_wgrad_kernel<32, false>);
  const size_t smem = pl[0] == 64 ? WgradTile<64>::smem : WgradTile<32>::smem;
  SIGMA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  void *args[] = {&p};
  SIGMA_CHECK_CUDA(cudaLaunchKernel(kern, dim3((unsigned)pl[1], (unsigned)pl[2]), dim3(WG_THREADS), args, smem, stream));
  count_launch();
  int rc = sum_parts_det_launch(p.part_w, p.nsplit, 9LL * Cout * Cin, 9LL * Cout * Cin, 0, dw, stream);
  if (rc) return rc;
  return db ? sum_parts_det_launch(p.part_b, p.nsplit, Cout, Cout, 0, db, stream) : SIGMA_OK;
}

}  // namespace sigma
