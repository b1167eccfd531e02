// Declarations shared between the library's translation units: every host function, kernel and parameter block that is
// used outside the file that defines it, declared once (default arguments included).  Each defining file includes this
// header (through common.cuh), so the compiler checks every definition against its declaration.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/sigma_b200.h"

namespace sigma {

// ---- parameter blocks ----
// Launch plan of one op-level scan sweep (scan_op*.cu): what the launcher runs and what sigma_test_scan_plan reports.
struct ScanOpPlan {
  int nsplit;            // L-segments
  int tiles_per_split;   // position tiles per segment
  int ntiles;            // position tiles of the sequence
  int DT;                // channels per CTA
  int nst;               // ring / pipeline stages
};

// Element code of e4m3 rows with one fp32 scale per row (the FP8 inference mode's row-norm output, E4M3Rows in common.cuh).
// Internal to the library: no entry point takes it, so it is not one of the public SIGMA_F32 / SIGMA_F16 / SIGMA_BF16 codes.
constexpr int SIGMA_E4M3_ROWS = 3;

// One row-norm launch.  The element types of y / z (input) and out are passed to row_norm_launch beside this block: the
// pointers are typed fp32 but hold elements of those types, and strides count them.  gamma, beta and gate are fp32.
struct RowNormParams {
  const float *y;          // K slabs
  long long k_stride;      // elements between slabs
  int K;
  const float *gamma, *beta;
  const float *z; long long z_row_stride;       // nullable
  const float *gate;                            // nullable, (rows / rows_per_batch, D)
  float *out;
  long long rows, rows_per_batch;
  long long in_batch_stride, out_batch_stride, out_row_stride;
  int D;
  float eps;
  // row addressing mode (fast kernel only): 0 = plain rows;
  // 1 = PatchMerging2D gather (vmamba.py:619-636): y is (batch, gH, gW, D/4), row (b,i,j) = the four pixels
  //     (2i,2j), (2i+1,2j), (2i,2j+1), (2i+1,2j+1) concatenated, zeros beyond odd gH / gW;
  // 2 = PatchExpand pixel shuffle (MambaDecoder.py:24-28): input rows are (b, h, w, p1, p2) sub-rows of D channels,
  //     row lands at out (b, 2h+p1, 2w+p2)
  int mode = 0, gH = 0, gW = 0;
  float *qscale = nullptr;   // e4m3 output: row r's scale
};

struct ImagePreParams {
  const unsigned char *src;   // (H0, W0, 3) uint8, HWC
  float *dst;                 // (3, OH, OW) float32 (one image of an NCHW batch)
  const unsigned char *lsrc;  // nullable: (H0, W0) uint8 labels
  long long *ldst;            // nullable: (OH, OW) int64 labels
  int H0, W0, SH, SW, OH, OW, off_y, off_x, mirror_src, mirror_out, label_pad;
  int clip_y0, clip_x0, clip_y1, clip_x1;   // only this rectangle of the scaled image is visible (a sliding window); rest = pad
  double scale_y, scale_x;    // source pixels per scaled pixel (cv2: 1/fy, 1/fx or H0/SH, W0/SW)
  double mean[3], stdv[3];
};

// ---- api.cu: host-side error state (thread-local string, no exceptions across the ABI) and the launch counter ----
void set_error(const char *fmt, ...);
void count_launch(int n = 1);

// ---- ss2d_scan_host.cu ----
// The one tensor-map encoder: cuTensorMapEncodeTiled resolved at run time through the runtime's driver entry point (the
// library does not link libcuda).  dims innermost first, strides_bytes for dims 1..rank-1; element strides 1, no interleave,
// no out-of-bounds fill.  Returns 0 or SIGMA_ECUDA with the library error string set.
int make_tmap(CUtensorMap *map, CUtensorMapDataType dtype, int rank, const void *base, const uint64_t *dims,
              const uint64_t *strides_bytes, const uint32_t *box, CUtensorMapSwizzle swz, CUtensorMapL2promotion promo);
int pad_rp(int R);   // dt_rank padded to an instantiated width (4, 8, 12, 16, 24, 32, 48, 64), -1 beyond 64
size_t ss2d_scan_workspace_bytes(int kind, int batch, int D, int N);
// xc_dtype: element type of xc and y, SIGMA_F32, SIGMA_BF16 or SIGMA_F16; dsave / hsave (training forward): delta' slabs and
// block-start states for the backward (with SIGMA_BF16 / SIGMA_F16: the bf16 / fp16 training modes, whose delta' slabs are 16-bit too)
int ss2d_scan_fwd(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                  const float *Ds, float *y, int batch, int H, int W, int D, int N, int R, int Cp, void *ws,
                  size_t ws_bytes, int force_split, cudaStream_t stream, float *dsave = nullptr, float *hsave = nullptr,
                  int xc_dtype = SIGMA_F32);
int ss2d_pick_segments_hook(long long ctas, int nw, int ntiles, int N);
int ss2d_fwd_plan_hook(int kind, int batch, int H, int W, int D, int N, int R, int xc_dtype, int force_split, size_t ws_bytes,
                       long long *out8);

// ---- ss2d_scan_bwd.cu ----
int ss2d_save_tiles(int kind, int H, int W);   // 16-position blocks of the longest walk
size_t ss2d_scan_hs_bytes(int kind, int batch, int H, int W, int D, int N);
size_t ss2d_scan_bwd_workspace_bytes(int kind, int batch, int H, int W, int D, int N);
size_t ss2d_scan_bwd_det_workspace_bytes(int kind, int batch, int H, int W, int D, int N);
int ss2d_bwd_plan_hook(int kind, int batch, int H, int W, int D, int N, int force_split, long long *out4);
// delta / hs: the delta' slabs and block-start states the training forward wrote; det: the deterministic build; xdtype
// SIGMA_BF16 / SIGMA_F16 (excludes det): xc, dy and delta are bf16 / fp16 behind the float pointers
int ss2d_scan_bwd(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A, const float *Ds,
                  const float *dy, const float *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl, float *dA, float *dDs,
                  float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *ws, size_t ws_bytes, int force_split,
                  cudaStream_t stream, int det = 0, int xdtype = SIGMA_F32);

// ---- scan_op.cu: generic op-level scan forward ----
__global__ void scan_combine_kernel(float *carry, long long nrows, int nsplit, int NP);
int scan_op_npad(int N);
size_t scan_op_workspace_bytes(int batch, int dim, int dstate);
ScanOpPlan scan_op_fwd_generic_plan(int batch, int dim, int L, int N, int G, bool have_ws, int force_split);
template <typename T>
int scan_op_fwd_generic(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                        const float *bias, void *out, float *x, float *hs, int batch, int dim, int L, int N, int G,
                        int softplus, const sigma_scan_strides &s, void *ws, size_t ws_bytes, int force_split,
                        cudaStream_t stream);

// ---- scan_op_tma.cu: TMA-staged op-level scan forward ----
cudaError_t prep_kernel_once(const void *fn);
int pick_segments(long long ctas_base, int ntiles, long long slots, double pass_factor, int max_split);
size_t scan_op_tma_workspace_bytes(int batch, int dim, int dstate);
ScanOpPlan scan_op_fwd_tma_plan(int elem_bytes, int batch, int dim, int L, int N, int G, bool have_ws, int force_split);
template <typename T>
bool scan_op_tma_eligible(const void *u, const void *delta, const void *B, const void *C, const void *out, int dim, int L,
                          int N, int G, const sigma_scan_strides &s);
template <typename T>
int scan_op_fwd_tma(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                    const float *bias, void *out, float *x, float *hs, int batch, int dim, int L, int N, int G, int softplus,
                    const sigma_scan_strides &s, void *ws, size_t ws_bytes, int force_split, cudaStream_t stream);

// ---- scan_op_bwd.cu: generic op-level scan backward ----
size_t scan_op_bwd_workspace_bytes(int batch, int dim, int L, int N, int elem_bytes);
size_t scan_op_bwd_det_bytes(int batch, int dim, int L, int N, int G);   // scratch of the deterministic build (det_ws)
template <typename T>
int scan_op_bwd_generic(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                        const float *bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                        float *dD, float *dbias, int batch, int dim, int L, int N, int G, int softplus, void *ws,
                        size_t ws_bytes, cudaStream_t stream, void *det_ws);

// ---- scan_op_bwd_tma.cu: TMA-staged op-level scan backward ----
__global__ void scan_combine_rev_kernel(float *carry, long long nrows, int nsplit, int NP);
size_t scan_op_bwd_tma_workspace_bytes(int batch, int dim, int L, int N, int elem_bytes);
size_t scan_op_bwd_tma_det_bytes(int batch, int dim, int L, int N, int G);   // scratch of the deterministic build (det_ws)
ScanOpPlan scan_op_bwd_tma_plan(int elem_bytes, int batch, int dim, int L, int N, int G, int force_split);
template <typename T>
int scan_op_bwd_tma(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                    const float *bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC, float *dD,
                    float *dbias, int batch, int dim, int L, int N, int G, int softplus, void *ws, size_t ws_bytes,
                    int force_split, cudaStream_t stream, void *det_ws);

// ---- scan_op_bwd_wide.cu: op-level scan backward for 16 < d_state <= 256 (deterministic, every entry point) ----
size_t scan_op_bwd_wide_workspace_bytes(int batch, int dim, int L, int N, int G);   // 0 for a call it does not take
ScanOpPlan scan_op_bwd_wide_plan(int L);
template <typename T>
int scan_op_bwd_wide(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D, const float *bias,
                     const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC, float *dD, float *dbias, int batch,
                     int dim, int L, int N, int G, int softplus, void *ws, size_t ws_bytes, cudaStream_t stream);

// ---- det_reduce.cu ----
int sum_parts_det_launch(const float *part, int nparts, long long ncols, long long inner, long long ostride, float *out, cudaStream_t stream);
int upsample_bilinear_bwd_launch(const float *dy, float *dx, int batch, int C, int Hin, int Win, int Hout, int Wout, float rh, float rw,
                                 int channels_last, cudaStream_t stream);

// ---- rowwise.cu ----
// ti: element type of y and z, to: of out.  The pairs with instances: (SIGMA_F32, SIGMA_F32 / SIGMA_BF16 / SIGMA_F16 /
// SIGMA_E4M3_ROWS), (SIGMA_BF16, SIGMA_BF16 / SIGMA_E4M3_ROWS) and (SIGMA_F16, SIGMA_F16); any other is SIGMA_EUNSUPPORTED.
int row_norm_launch(int ti, int to, const RowNormParams &p, cudaStream_t stream);
int quantize_e4m3_rows_launch(const void *x, bool bf16, long long ldx, void *q, long long ldq, float *scale, long long rows, int C,
                              cudaStream_t stream);
// dtype: element type of x, dy and dx, SIGMA_F32, SIGMA_BF16 or SIGMA_F16; part != nullptr (SIGMA_F32 only): the deterministic
// build (layernorm_bwd_det_workspace_bytes of scratch)
int layernorm_bwd_launch(int dtype, const void *x, const void *dy, const float *gamma, void *dx, float *dgamma, float *dbeta,
                         long long rows, int D, float eps, cudaStream_t stream, float *part = nullptr);
size_t layernorm_bwd_det_workspace_bytes(long long rows, int D);
int upsample2x_norm_launch(const float *in, const float *gamma, const float *beta, const float *wcls, int ncls, float *out,
                           int B, int Hin, int Win, int C, float eps, cudaStream_t stream);
int pool_avgmax_partial_launch(const float *x, float *partial, int B, long long L, int C, int nslice, cudaStream_t stream);
int scale_add_launch(const float *a, const float *sa, const float *b, const float *sb, float *out, long long rows,
                     long long rows_per_batch, int C, cudaStream_t stream);

// ---- dwconv_tma.cu ----
// dtype SIGMA_F32, SIGMA_BF16 or SIGMA_F16 x and y; x 16-byte aligned with strides multiples of 16 bytes (TMA: the caller checks)
int dwconv3x3_silu_fwd_launch(int dtype, const void *x, long long x_row_stride, long long x_batch_stride, const float *w,
                              const float *bias, void *y, long long y_batch_stride, int batch, int H, int W, int D, cudaStream_t stream);
// backward: dtype SIGMA_F32, SIGMA_BF16 or SIGMA_F16 x, dy and dx; ws holds dwconv3x3_silu_bwd_workspace_bytes (16-byte aligned)
size_t dwconv3x3_silu_bwd_workspace_bytes(int batch, int H, int W, int D);
int dwconv3x3_silu_bwd_launch(int dtype, const void *x, long long x_row_stride, long long x_batch_stride, const float *w,
                              const float *bias, const void *dy, long long dy_batch_stride, void *dx, long long dx_batch_stride, float *dw,
                              float *db, int batch, int H, int W, int D, void *ws, cudaStream_t stream);

// ---- gemm_tf32.cu ----
// The operand kind of the wgmma GEMM: fp32 operands read as TF32 or split into tf32x3 (A·W = A_hi·W_hi + A_lo·W_hi + A_hi·W_lo),
// bf16, fp16 or e4m3 operands; fp32 accumulation in every case
enum class GemmOp { TF32, TF32X3, BF16, F16, E4M3 };
// C = A (M, K) · W (N, K)^T (+ bias) (+ residual · rscale), lda / ldc / ldr in elements.  TF32X3: W = W_hi and W_lo, output tiles
// stored with TMA unless reg_epilogue (the TMA-stored epilogue's reference in the tests, sigma_test_linear_tf32x3_regs); C and
// the residual then need 16-byte-aligned bases and row strides (sigma_linear_tf32x3 checks it).  E4M3: A and W scaled by the fp32
// sa (M) and sw (N) before the bias.  c_16 = 1: C stored as fp16 (F16) or bf16 (BF16, E4M3), else fp32; bias / residual / rscale
// are fp32 for every kind.
int gemm_launch(GemmOp op, const void *A, long long lda, const void *W, const void *W_lo, const float *sa, const float *sw,
                const float *bias, const float *residual, long long ldr, const float *rscale, void *C, long long ldc, int c_16,
                long long M, int N, int K, cudaStream_t stream, bool reg_epilogue = false);
// epi 1 (with act 1): also store pre = conv + bias to aux; epi 2 (act 0): multiply the result by GELU'(aux) (aux in y's layout)
int conv3x3_tf32_launch(const float *x, const float *W9, const float *W9_lo, const float *bias, int act, float *y, int B, int H, int W,
                        int Cin, int Cout, cudaStream_t stream, int epi = 0, float *aux = nullptr);
int conv3x3_pitched_launch(const float *x, long long x_ld, const float *W9, const float *W9_lo, long long w_ld, const float *bias, int act,
                           float *y, long long y_ld, int B, int H, int W, int Cin, int Cout, cudaStream_t stream, int epi = 0,
                           float *aux = nullptr);
int split_tf32_launch(const float *x, float *hi, float *lo, long long n, cudaStream_t stream);
int gemm_pick_bn_hook(int N, long long m_tiles);
int gemm_plan_hook(long long M, int N, int K, int mode, int conv_B, int conv_H, int conv_W, long long *out);

// ---- conv3x3_wgrad.cu ----
// Launch plan of the weight gradient: {output channels per tile, output tiles, partial rows, CTAs}
void conv3x3_wgrad_plan(int batch, int H, int W, int Cin, int Cout, long long *out4);
size_t conv3x3_wgrad_workspace_bytes(int batch, int H, int W, int Cin, int Cout);
// x_ld > 0: x and dy rows are x_ld / dy_ld elements apart (cab_wgrad_pitched_kernel); 0: Cin / Cout (conv3x3_wgrad_kernel)
int conv3x3_wgrad_launch(const float *x, int gelu_x, const float *dy, float *dw, float *db, int batch, int H, int W, int Cin, int Cout,
                         int x3, void *ws, cudaStream_t stream, int x_ld = 0, int dy_ld = 0);

// ---- evaluator.cu ----
int argmax_hist_launch(const float *logits, const void *labels, int label_bytes, unsigned long long *hist,
                       unsigned long long *counts, unsigned char *pred_out, int batch, int ncls, long long HW, cudaStream_t stream);
int image_pre_launch(const ImagePreParams &p, cudaStream_t stream);
int eval_exp_accumulate_launch(const float *logits, const float *logits_flip, float *acc, int ncls, int TH, int TW, int m_top, int m_left,
                               int vh, int vw, int AH, int AW, int ay, int ax, cudaStream_t stream);
int eval_resize_add_launch(const float *acc, int ncls, int AH, int AW, int m_top, int m_left, int SH, int SW, double *out, int H0, int W0,
                           cudaStream_t stream);
int eval_argmax_hist_launch(const double *score, const unsigned char *labels, unsigned char *pred, unsigned long long *hist,
                            unsigned long long *counts, int ncls, long long HW, cudaStream_t stream);

}  // namespace sigma
