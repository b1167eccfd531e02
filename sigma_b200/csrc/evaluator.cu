// SURVEY.md §8(f) rank 2 — the evaluator's per-image metric on the device (eval.py:22-29, utils/metric.py:8-15):
//   pred = argmax_c logits[b, c, h, w]   (the reference takes argmax of exp(score): same index; first maximum on ties,
//                                          as numpy.argmax)
//   k = label in [0, ncls);  hist[label·ncls + pred] += 1;  labeled += 1;  correct += (pred == label)
// so only ncls² + 2 integers leave the GPU instead of the logits.  Integer work, bit-exact against the reference's numpy.
// One thread per pixel (coalesced over w for every class plane), shared-memory histogram per CTA, 64-bit global atomics.
#include <algorithm>

#include "common.cuh"

namespace sigma {

template <typename LabelT>
__global__ void __launch_bounds__(256) argmax_hist_kernel(const float *__restrict__ logits, const LabelT *__restrict__ labels,
                                                         unsigned long long *__restrict__ hist, unsigned long long *__restrict__ counts,
                                                         unsigned char *__restrict__ pred_out, int batch, int ncls, long long HW) {
  extern __shared__ unsigned int sh[];   // ncls*ncls bins + labeled + correct
  const int nb = ncls * ncls;
  for (int i = threadIdx.x; i < nb + 2; i += blockDim.x) sh[i] = 0u;
  __syncthreads();
  const long long total = (long long)batch * HW;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const long long b = p / HW, r = p - b * HW;
    const float *lp = logits + b * ncls * HW + r;
    float best = lp[0];
    int arg = 0;
    for (int c = 1; c < ncls; ++c) {
      const float v = __ldg(lp + (long long)c * HW);
      if (v > best) { best = v; arg = c; }          // strict: the first maximum wins (numpy.argmax)
    }
    if (pred_out) pred_out[p] = (unsigned char)arg;
    const long long g = (long long)labels[p];
    if (g >= 0 && g < ncls) {
      atomicAdd(&sh[(int)g * ncls + arg], 1u);
      atomicAdd(&sh[nb], 1u);
      if (arg == (int)g) atomicAdd(&sh[nb + 1], 1u);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nb; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[i], (unsigned long long)sh[i]);
  if (threadIdx.x == 0) {
    if (sh[nb]) atomicAdd(&counts[0], (unsigned long long)sh[nb]);
    if (sh[nb + 1]) atomicAdd(&counts[1], (unsigned long long)sh[nb + 1]);
  }
}

int argmax_hist_launch(const float *logits, const void *labels, int label_bytes, unsigned long long *hist,
                       unsigned long long *counts, unsigned char *pred_out, int batch, int ncls, long long HW, cudaStream_t stream) {
  const long long total = (long long)batch * HW;
  if (total == 0) return SIGMA_OK;
  // a CTA's shared counters are 32-bit: bound the pixels per CTA below 2^32 (grid-stride over <= kNumSMs*8 CTAs)
  const unsigned grid = (unsigned)std::min<long long>((total + 255) / 256, kNumSMs * 8);
  const size_t smem = (size_t)(ncls * ncls + 2) * sizeof(unsigned int);
  if (smem > 227 * 1024) { set_error("sigma_argmax_hist_fwd: num_classes=%d: the per-CTA histogram (%zu B) exceeds shared memory (max 238 classes)", ncls, smem); return SIGMA_EINVAL; }
  if (smem > 48 * 1024) {   // > 110 classes: opt in to large dynamic shared memory
    SIGMA_CHECK_CUDA(cudaFuncSetAttribute(argmax_hist_kernel<unsigned char>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SIGMA_CHECK_CUDA(cudaFuncSetAttribute(argmax_hist_kernel<int>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    SIGMA_CHECK_CUDA(cudaFuncSetAttribute(argmax_hist_kernel<long long>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  if (label_bytes == 1)
    argmax_hist_kernel<unsigned char><<<grid, 256, smem, stream>>>(logits, (const unsigned char *)labels, hist, counts, pred_out, batch, ncls, HW);
  else if (label_bytes == 4)
    argmax_hist_kernel<int><<<grid, 256, smem, stream>>>(logits, (const int *)labels, hist, counts, pred_out, batch, ncls, HW);
  else if (label_bytes == 8)
    argmax_hist_kernel<long long><<<grid, 256, smem, stream>>>(logits, (const long long *)labels, hist, counts, pred_out, batch, ncls, HW);
  else { set_error("sigma_argmax_hist_fwd: label_bytes=%d unsupported (1, 4, 8)", label_bytes); return SIGMA_EINVAL; }
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// Either side of the hot path (SURVEY.md §8f ranks 2 and 3): the evaluator's per-image pipeline
// (engine/evaluator.py:433-522) and the train / eval pre-processing (dataloader/dataloader.py:8-50,
// utils/transforms.py:61-75,182-187) on the device, so the model's inputs never exist on the host as float tensors and
// its score maps never leave HBM.
// ---------------------------------------------------------------------------------------------------------------------

// cv2.resize(INTER_LINEAR) on 8-bit images, generic (non-IPP) path: 11-bit fixed-point coefficients
// (INTER_RESIZE_COEF_BITS), horizontal pass to 32-bit ints, vertical pass with the >>4 / >>16 / +2 >>2 rounding of
// VResizeLinear<uchar>.  f = (float)((d + 0.5)·scale − 0.5), clamped at the borders like resizeGeneric_.
struct Lin8u { int i0, i1, a0, a1; };
__device__ __forceinline__ Lin8u lin8u_coef(int d, int sn, double scale) {
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f -= (float)s;
  if (s < 0) { s = 0; f = 0.f; }
  if (s >= sn - 1) { s = sn - 1; f = 0.f; }
  Lin8u c;
  c.i0 = s; c.i1 = min(s + 1, sn - 1);
  c.a0 = __float2int_rn((1.f - f) * 2048.f);
  c.a1 = __float2int_rn(f * 2048.f);
  return c;
}

// One output pixel per thread: out(c, oy, ox) = pad 0 outside the scaled image, else ((resized / 255) − mean) / std in
// double like utils/transforms.py:182-187, rounded to float like np.ascontiguousarray(..., dtype=float32).
__global__ void __launch_bounds__(256) image_pre_kernel(const ImagePreParams p) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)p.OH * p.OW) return;
  const int oy = (int)(idx / p.OW), oxo = (int)(idx - (long long)oy * p.OW);
  const int ox = p.mirror_out ? p.OW - 1 - oxo : oxo;          // evaluator.py:512-515: flip of the padded network input
  const int sy = oy + p.off_y, sx = ox + p.off_x;
  const bool inside = sy >= p.clip_y0 && sy < p.clip_y1 && sx >= p.clip_x0 && sx < p.clip_x1;
  float v[3] = {0.f, 0.f, 0.f};
  long long lab = p.label_pad;
  if (inside) {
    const bool same = p.SH == p.H0 && p.SW == p.W0;
    const Lin8u cy = same ? Lin8u{sy, sy, 2048, 0} : lin8u_coef(sy, p.H0, p.scale_y);
    const Lin8u cx = same ? Lin8u{sx, sx, 2048, 0} : lin8u_coef(sx, p.W0, p.scale_x);
    const int x0 = p.mirror_src ? p.W0 - 1 - cx.i0 : cx.i0, x1 = p.mirror_src ? p.W0 - 1 - cx.i1 : cx.i1;   // cv2.flip(img, 1) first
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int s00 = p.src[((long long)cy.i0 * p.W0 + x0) * 3 + c], s01 = p.src[((long long)cy.i0 * p.W0 + x1) * 3 + c];
      const int s10 = p.src[((long long)cy.i1 * p.W0 + x0) * 3 + c], s11 = p.src[((long long)cy.i1 * p.W0 + x1) * 3 + c];
      const int r0 = s00 * cx.a0 + s01 * cx.a1, r1 = s10 * cx.a0 + s11 * cx.a1;
      const int px = (((cy.a0 * (r0 >> 4)) >> 16) + ((cy.a1 * (r1 >> 4)) >> 16) + 2) >> 2;
      v[c] = (float)((((double)px / 255.0) - p.mean[c]) / p.stdv[c]);
    }
    if (p.lsrc) {   // labels: cv2.INTER_NEAREST (dataloader.py:21): src = min(floor(d·scale), n−1)
      const int ly = same ? sy : min((int)floor((double)sy * p.scale_y), p.H0 - 1);
      int lx = same ? sx : min((int)floor((double)sx * p.scale_x), p.W0 - 1);
      if (p.mirror_src) lx = p.W0 - 1 - lx;
      lab = p.lsrc[(long long)ly * p.W0 + lx];
    }
  }
  const long long o = (long long)oy * p.OW + oxo, plane = (long long)p.OH * p.OW;
  p.dst[o] = v[0]; p.dst[plane + o] = v[1]; p.dst[2 * plane + o] = v[2];
  if (p.ldst) p.ldst[o] = lab;
}

int image_pre_launch(const ImagePreParams &p, cudaStream_t stream) {
  const long long total = (long long)p.OH * p.OW;
  if (total == 0) return SIGMA_OK;
  image_pre_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(p);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

// evaluator.py:505-520 + 481-488: score = exp(logits (+ flip(logits of the flipped input))), margins cropped, added into the
// window's place of the scale's score map  acc (ncls, AH, AW) float32.
__global__ void __launch_bounds__(256) eval_exp_accumulate_kernel(const float *__restrict__ logits, const float *__restrict__ logits_flip,
                                                                  float *__restrict__ acc, int ncls, int TH, int TW, int m_top,
                                                                  int m_left, int vh, int vw, int AH, int AW, int ay, int ax) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)ncls * vh * vw) return;
  const int x = (int)(idx % vw), y = (int)((idx / vw) % vh), c = (int)(idx / ((long long)vw * vh));
  const int ty = y + m_top, tx = x + m_left;
  float s = logits[((long long)c * TH + ty) * TW + tx];
  if (logits_flip) s += logits_flip[((long long)c * TH + ty) * TW + (TW - 1 - tx)];
  acc[((long long)c * AH + ay + y) * AW + ax + x] += expf(s);
}

// evaluator.py:497-499 + 447-448: processed_pred (H0, W0, ncls) float64 += cv2.resize(score.permute(1,2,0) [margin cropped],
// (W0, H0), INTER_LINEAR) — the float path of cv2 (float coefficients, horizontal then vertical).
__global__ void __launch_bounds__(256) eval_resize_add_kernel(const float *__restrict__ acc, int ncls, int AH, int AW, int m_top, int m_left,
                                                              int SH, int SW, double *__restrict__ out, int H0, int W0) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)H0 * W0) return;
  const int dy = (int)(idx / W0), dx = (int)(idx - (long long)dy * W0);
  const bool same = SH == H0 && SW == W0;
  float fy = 0.f, fx = 0.f;
  int sy = dy, sx = dx;
  if (!same) {
    fy = (float)(((double)dy + 0.5) * ((double)SH / H0) - 0.5); sy = (int)floorf(fy); fy -= (float)sy;
    if (sy < 0) { sy = 0; fy = 0.f; }
    if (sy >= SH - 1) { sy = SH - 1; fy = 0.f; }
    fx = (float)(((double)dx + 0.5) * ((double)SW / W0) - 0.5); sx = (int)floorf(fx); fx -= (float)sx;
    if (sx < 0) { sx = 0; fx = 0.f; }
    if (sx >= SW - 1) { sx = SW - 1; fx = 0.f; }
  }
  const int sy1 = min(sy + 1, SH - 1), sx1 = min(sx + 1, SW - 1);
  for (int c = 0; c < ncls; ++c) {
    const float *pl = acc + (long long)c * AH * AW;
    float v;
    if (same) {
      v = pl[(long long)(m_top + sy) * AW + m_left + sx];
    } else {
      const float r0 = __fadd_rn(__fmul_rn(pl[(long long)(m_top + sy) * AW + m_left + sx], 1.f - fx), __fmul_rn(pl[(long long)(m_top + sy) * AW + m_left + sx1], fx));
      const float r1 = __fadd_rn(__fmul_rn(pl[(long long)(m_top + sy1) * AW + m_left + sx], 1.f - fx), __fmul_rn(pl[(long long)(m_top + sy1) * AW + m_left + sx1], fx));
      v = __fadd_rn(__fmul_rn(r0, 1.f - fy), __fmul_rn(r1, fy));
    }
    out[idx * ncls + c] += (double)v;
  }
}

// evaluator.py:451: pred = processed_pred.argmax(2) (first maximum), then utils/metric.py:8-15 on the device
__global__ void __launch_bounds__(256) eval_argmax_hist_kernel(const double *__restrict__ score, const unsigned char *__restrict__ labels,
                                                               unsigned char *__restrict__ pred, unsigned long long *__restrict__ hist,
                                                               unsigned long long *__restrict__ counts, int ncls, long long HW) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= HW) return;
  const double *sp = score + idx * ncls;
  double best = sp[0];
  int arg = 0;
  for (int c = 1; c < ncls; ++c)
    if (sp[c] > best) { best = sp[c]; arg = c; }
  pred[idx] = (unsigned char)arg;
  if (labels) {
    const int g = labels[idx];
    if (g < ncls) {
      atomicAdd(&hist[(long long)g * ncls + arg], 1ull);
      atomicAdd(&counts[0], 1ull);
      if (g == arg) atomicAdd(&counts[1], 1ull);
    }
  }
}

int eval_exp_accumulate_launch(const float *logits, const float *logits_flip, float *acc, int ncls, int TH, int TW, int m_top, int m_left,
                               int vh, int vw, int AH, int AW, int ay, int ax, cudaStream_t stream) {
  const long long total = (long long)ncls * vh * vw;
  if (total == 0) return SIGMA_OK;
  eval_exp_accumulate_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(logits, logits_flip, acc, ncls, TH, TW, m_top, m_left, vh, vw,
                                                                                   AH, AW, ay, ax);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}
int eval_resize_add_launch(const float *acc, int ncls, int AH, int AW, int m_top, int m_left, int SH, int SW, double *out, int H0, int W0,
                           cudaStream_t stream) {
  const long long total = (long long)H0 * W0;
  eval_resize_add_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(acc, ncls, AH, AW, m_top, m_left, SH, SW, out, H0, W0);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}
int eval_argmax_hist_launch(const double *score, const unsigned char *labels, unsigned char *pred, unsigned long long *hist,
                            unsigned long long *counts, int ncls, long long HW, cudaStream_t stream) {
  eval_argmax_hist_kernel<<<(unsigned)((HW + 255) / 256), 256, 0, stream>>>(score, labels, pred, hist, counts, ncls, HW);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

}  // namespace sigma
