// Deterministic training kernels (torch.use_deterministic_algorithms): the fixed-order sum that replaces the float atomics
// of the backward kernels, and the gather-form backward of bilinear upsampling.
//
// Every `_det` backward writes one partial per contributor (channel tile, image, L-segment, warp) into a workspace
// instead of adding into its output; sum_parts_det_kernel then adds the partials of every output element in an order fixed
// by the launch plan alone, so the same inputs and plan give the same bits whatever the CTA schedule.
#include <algorithm>

#include "common.cuh"

namespace sigma {

// out[(c / inner) * ostride + c % inner] = sum over p of part[p * ncols + c].  Block (32, S): lane x owns a column, row y
// sums the parts y, y + S, y + 2S, ... in ascending order, then row 0 adds the S row sums in ascending y.
__global__ void __launch_bounds__(256) sum_parts_det_kernel(const float *__restrict__ part, int nparts, long long ncols, long long inner,
                                                            long long ostride, float *__restrict__ out) {
  __shared__ float rs[8][32];
  const int S = blockDim.y, x = threadIdx.x, y = threadIdx.y;
  const long long c = (long long)blockIdx.x * 32 + x;
  float acc = 0.f;
  if (c < ncols)
    for (int pi = y; pi < nparts; pi += S) acc += part[(long long)pi * ncols + c];
  rs[y][x] = acc;
  __syncthreads();
  if (y == 0 && c < ncols) {
    float s = rs[0][x];
    for (int j = 1; j < S; ++j) s += rs[j][x];
    out[(c / inner) * ostride + c % inner] = s;
  }
}

int sum_parts_det_launch(const float *part, int nparts, long long ncols, long long inner, long long ostride, float *out, cudaStream_t stream) {
  if (ncols <= 0) return SIGMA_OK;
  const int S = nparts < 8 ? (nparts < 1 ? 1 : nparts) : 8;
  const long long nb = (ncols + 31) / 32;
  if (nb > 0x7fffffffLL) { set_error("sum_parts_det: %lld columns is too many", ncols); return SIGMA_EINVAL; }
  sum_parts_det_kernel<<<(unsigned)nb, dim3(32, S), 0, stream>>>(part, nparts, ncols, inner, ostride, out);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

// ---- backward of F.interpolate(mode="bilinear", align_corners=False) ----
// torch's source-index rule (aten/src/ATen/native/UpSample.h: area_pixel_compute_source_index, align_corners = false):
// src = max(ratio·(o + 0.5) − 0.5, 0) in fp32, i0 = (int)src, i1 = i0 + (i0 < in − 1), lambda1 = src − i0, lambda0 = 1 − lambda1.
// The ratio is 1/scale_factor when the caller gave one, in/out otherwise (computed on the host, rounded to fp32 as torch does).
__device__ __forceinline__ float up_tap_weight(float ratio, int o, int in, int i) {
  float src = ratio * ((float)o + 0.5f) - 0.5f;
  src = src < 0.f ? 0.f : src;
  const int i0 = (int)src, i1 = i0 + (i0 < in - 1 ? 1 : 0);
  const float l1 = src - (float)i0, l0 = 1.f - l1;
  return (i0 == i ? l0 : 0.f) + (i1 == i ? l1 : 0.f);
}

__device__ __forceinline__ void up_range(float ratio, int i, int out, int &lo, int &hi) {
  // outputs whose source lies in (i - 1, i + 1): o in ((i - 0.5) / ratio - 0.5, (i + 1.5) / ratio - 0.5), widened by 2
  lo = max(0, (int)floorf(((float)i - 0.5f) / ratio - 0.5f) - 2);
  hi = min(out - 1, (int)ceilf(((float)i + 1.5f) / ratio - 0.5f) + 2);
}

// One thread per input element (n, c, h, w); dx = sum over the output rows oh (ascending) and columns ow (ascending) that
// tap it of weight_h(oh)·weight_w(ow)·dy[n, c, oh, ow].  CL: channels-last element order (c fastest), else NCHW.
template <bool CL>
__global__ void __launch_bounds__(256) upsample_bilinear_bwd_det_kernel(const float *__restrict__ dy, float *__restrict__ dx, int batch,
                                                                        int C, int Hin, int Win, int Hout, int Wout, float rh, float rw) {
  const long long total = (long long)batch * C * Hin * Win;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    int n, c, h, w;
    long long r = idx;
    if (CL) {
      c = (int)(r % C); r /= C; w = (int)(r % Win); r /= Win; h = (int)(r % Hin); n = (int)(r / Hin);
    } else {
      w = (int)(r % Win); r /= Win; h = (int)(r % Hin); r /= Hin; c = (int)(r % C); n = (int)(r / C);
    }
    const long long sH = CL ? (long long)Wout * C : Wout, sW = CL ? C : 1;
    const float *g = dy + (CL ? (long long)n * Hout * Wout * C + c : ((long long)n * C + c) * Hout * Wout);
    int oh0, oh1, ow0, ow1;
    up_range(rh, h, Hout, oh0, oh1);
    up_range(rw, w, Wout, ow0, ow1);
    float acc = 0.f;
    for (int oh = oh0; oh <= oh1; ++oh) {
      const float wh = up_tap_weight(rh, oh, Hin, h);
      if (wh == 0.f) continue;
      for (int ow = ow0; ow <= ow1; ++ow) {
        const float ww = up_tap_weight(rw, ow, Win, w);
        if (ww == 0.f) continue;
        acc = fmaf(wh * ww, g[oh * sH + ow * sW], acc);
      }
    }
    dx[idx] = acc;
  }
}

int upsample_bilinear_bwd_launch(const float *dy, float *dx, int batch, int C, int Hin, int Win, int Hout, int Wout, float rh, float rw,
                                 int channels_last, cudaStream_t stream) {
  const long long total = (long long)batch * C * Hin * Win;
  if (total == 0) return SIGMA_OK;
  const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, (long long)kNumSMs * 16);
  if (channels_last) upsample_bilinear_bwd_det_kernel<true><<<grid, 256, 0, stream>>>(dy, dx, batch, C, Hin, Win, Hout, Wout, rh, rw);
  else upsample_bilinear_bwd_det_kernel<false><<<grid, 256, 0, stream>>>(dy, dx, batch, C, Hin, Win, Hout, Wout, rh, rw);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

}  // namespace sigma
