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
  int x_ld, dy_ld;          // cab_wgrad_pitched_kernel: the row pitches of x and dy in elements (multiples of 4, >= Cin / Cout)
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

#define SIGMA_WGRAD_KERNEL conv3x3_wgrad_kernel
#define SIGMA_WGRAD_X_LD p.Cin
#define SIGMA_WGRAD_DY_LD p.Cout
#include "conv3x3_wgrad_kernel.inc"
#undef SIGMA_WGRAD_KERNEL
#undef SIGMA_WGRAD_X_LD
#undef SIGMA_WGRAD_DY_LD

// The same on pitched rows (the CAB convs of Sigma-base): x and dy rows are p.x_ld / p.dy_ld elements apart, and Cin, Cout need not
// be multiples of 4.  A chunk is staged when it starts below the count, and the pitch (a multiple of 4) keeps it inside the row, so a
// chunk that straddles the count also stages pad elements.  Those are input channels ci >= Cin (A rows, reaching only dW[., ci])
// and output channels co >= Cout (B columns, reaching only dW[co, .] and db[co]), none of which is stored: whatever the pads hold,
// no kept output sees it.
#define SIGMA_WGRAD_KERNEL cab_wgrad_pitched_kernel
#define SIGMA_WGRAD_X_LD p.x_ld
#define SIGMA_WGRAD_DY_LD p.dy_ld
#include "conv3x3_wgrad_kernel.inc"
#undef SIGMA_WGRAD_KERNEL
#undef SIGMA_WGRAD_X_LD
#undef SIGMA_WGRAD_DY_LD

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
                         int x3, void *ws, cudaStream_t stream, int x_ld, int dy_ld) {
  const bool pitched = x_ld > 0;
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
  p.x_ld = pitched ? x_ld : Cin; p.dy_ld = pitched ? dy_ld : Cout;
  const void *kern;
  if (pitched)
    kern = pl[0] == 64 ? (x3 ? (const void *)cab_wgrad_pitched_kernel<64, true> : (const void *)cab_wgrad_pitched_kernel<64, false>)
                       : (x3 ? (const void *)cab_wgrad_pitched_kernel<32, true> : (const void *)cab_wgrad_pitched_kernel<32, false>);
  else
    kern = pl[0] == 64 ? (x3 ? (const void *)conv3x3_wgrad_kernel<64, true> : (const void *)conv3x3_wgrad_kernel<64, false>)
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
