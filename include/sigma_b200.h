/*
 * sigma_b200 — C-ABI of the H100-native (sm_90a) SS2D / selective-scan hot path.
 *
 * Plain pointers and sizes only (no torch types).  Every pointer is a DEVICE pointer unless the
 * name ends in `_host`.  Every function launches on `stream` (a cudaStream_t passed as void*),
 * never synchronises, allocates nothing (scratch comes from the caller through `workspace`),
 * and returns 0 on success or a negative SIGMA_E* code; sigma_last_error() then holds a
 * human-readable message (thread-local).  No exceptions cross this boundary.
 *
 * The reference interface each entry point replaces is cited as file:line relative to the
 * reference repository (zifuwan/Sigma @ 5c619c6).  INTEGRATION.md shows the binding a
 * maintainer of the reference would add.
 */
#ifndef SIGMA_B200_H_
#define SIGMA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SIGMA_OK 0
#define SIGMA_EINVAL (-1)   /* bad shape / stride / dtype / null pointer            */
#define SIGMA_ECUDA (-2)    /* CUDA runtime or driver error (launch, tensor map...) */
#define SIGMA_EWORKSPACE (-3) /* workspace missing or too small                      */
#define SIGMA_EUNSUPPORTED (-4)

/* element types of u / delta / B / C / out (A, D, delta_bias and all states are fp32,
 * selective_scan.cpp:175-180) */
#define SIGMA_F32 0
#define SIGMA_F16 1
#define SIGMA_BF16 2

int sigma_abi_version(void);
const char *sigma_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py: gpu_launches) */
uint64_t sigma_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * a1. selective scan, op level.
 * Replaces `selective_scan_cuda_core.fwd(u, delta, A, B, C, D, delta_bias, delta_softplus,
 * nrows) -> [out, x]`  (csrc/selective_scan/selective_scan.cpp:165-249, kernel
 * selective_scan_fwd_kernel.cuh:64-206).
 *
 *   delta' = softplus?(delta + delta_bias[d]);  h[n,l] = exp(delta'·A[d,n])·h[n,l-1] + delta'·B[g,n,l]·u[l]
 *   out[d,l] = D[d]·u[l] + Σ_n C[g,n,l]·h[n,l],   g = d / (dim / ngroups)
 *
 * Layout: u, delta, out (batch, dim, seqlen) with unit stride along seqlen and the element
 * strides given below; A (dim, dstate) any strides; B, C (batch, ngroups, dstate, seqlen) unit
 * stride along seqlen.  `x` (nullable) receives the chunk-end states
 * (batch, dim, ceil(seqlen/2048), 2·dstate) fp32, interleaved (prod a, h), contiguous
 * (selective_scan.cpp:228, fwd_kernel.cuh:181-184; the first component is the running product since the START of the
 * sequence, as the reference's prefix callback keeps it).  D and delta_bias are nullable.  fp16 / bf16 are read and
 * written natively.  Calls whose rows are 16-byte aligned, whose channel groups are multiples of 32 and d_state in
 * {4, 8, 16} (every Sigma call) run the TMA-staged kernel (csrc/scan_op_tma.cu); anything else the generic one.
 * `workspace` only holds the L-segment carries (sigma_scan_fwd_workspace_bytes); without it the scan runs unsplit.
 * ------------------------------------------------------------------------------------------ */
typedef struct sigma_scan_strides {
  int64_t u_batch, u_dim;
  int64_t delta_batch, delta_dim;
  int64_t A_dim, A_dstate;
  int64_t B_batch, B_group, B_dstate;
  int64_t C_batch, C_group, C_dstate;
  int64_t out_batch, out_dim;
} sigma_scan_strides;

size_t sigma_scan_fwd_workspace_bytes(int batch, int dim, int seqlen, int dstate, int ngroups,
                                      int dtype);

int sigma_scan_fwd(const void *u, const void *delta, const float *A, const void *B, const void *C,
                   const float *D, const float *delta_bias, void *out, float *x,
                   int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                   int delta_softplus, const sigma_scan_strides *strides,
                   void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------
 * a3. backward of a1.
 * Replaces `selective_scan_cuda_core.bwd(u, delta, A, B, C, D, delta_bias, dout, x,
 * delta_softplus, nrows) -> [du, ddelta, dA, dB, dC, dD, ddelta_bias]`
 * (selective_scan.cpp:251-362, selective_scan_bwd_kernel.cuh:68-274).
 * All tensors contiguous, d_state <= 256, fp16 / bf16 natively.  `workspace` holds the forward states of the recompute sweep
 * (one every 16 positions) and the L-segment carries of both directions;  for 16 < d_state <= 256 ONE deterministic kernel
 * (no float atomics; csrc/scan_op_bwd_wide.cu) serves sigma_scan_bwd, sigma_scan_bwd_split and sigma_scan_bwd_det alike: no
 * L-segments (nsplit has no effect), the same bits from all three, and the workspace (the same size from both queries) holds
 * the states at every 32-position tile and the partial sums;
 * the reference's `x` is not needed.  du, ddelta: (batch, dim, seqlen) in `dtype`; dA (dim, dstate),
 * dD, ddelta_bias (dim) fp32 — OVERWRITTEN (not accumulated); dB, dC (batch, ngroups, dstate,
 * seqlen) fp32, overwritten.  dD / ddelta_bias may be NULL when D / delta_bias are NULL.
 * ------------------------------------------------------------------------------------------ */
size_t sigma_scan_bwd_workspace_bytes(int batch, int dim, int seqlen, int dstate, int ngroups, int dtype);

int sigma_scan_bwd(const void *u, const void *delta, const float *A, const void *B, const void *C,
                   const float *D, const float *delta_bias, const void *dout,
                   void *du, void *ddelta, float *dA, float *dB, float *dC, float *dD,
                   float *ddelta_bias,
                   int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                   int delta_softplus, void *workspace, size_t workspace_bytes, void *stream);

/* Deterministic build of sigma_scan_bwd (torch.use_deterministic_algorithms): the same outputs, bitwise reproducible for the
 * same inputs, GPU model and L-segment plan.  dB / dC are kept per channel tile of a group and dA / dD / ddelta_bias per
 * (batch, L-segment) in the workspace, then summed in a fixed order; no float atomics.  nsplit = 0 lets the library choose
 * the L-segments, as sigma_scan_bwd does. */
size_t sigma_scan_bwd_det_workspace_bytes(int batch, int dim, int seqlen, int dstate, int ngroups, int dtype);
int sigma_scan_bwd_det(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                       const float *delta_bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                       float *dD, float *ddelta_bias, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                       int delta_softplus, void *workspace, size_t workspace_bytes, int nsplit, void *stream);

/* ------------------------------------------------------------------------------------------
 * a4+a5 (+a8/a9 cores). Fused multi-direction SS2D scan, channels-last.
 * Replaces, in one launch, CrossScan (vmamba.py:80-98) + the dt_proj einsum (vmamba.py:199) +
 * delta_bias/softplus + SelectiveScan (vmamba.py:213) + the un-flip / un-transpose half of
 * CrossMerge (vmamba.py:100-108) of `cross_selective_scan` (vmamba.py:165-226); with
 * kind=SIGMA_DIRS_SEQ2 the K=2 core of `cross_selective_scan_multimodal_k2` (vmamba.py:369-430)
 * and with kind=SIGMA_DIRS_CROSS the two C-swapped scans of Cross_Mamba_Attention_SSM.forward
 * (vmamba.py:1528-1539).
 *
 *   xc    (batch, Lseq, D)          fp32, channels-last: the dwconv+SiLU output.  Lseq = H·W; for
 *                                   SEQ2 Lseq = 2·H·W = [rgb ‖ x] per image; for CROSS batch = 2·images,
 *                                   modality-major: [0, batch/2) rgb, [batch/2, batch) modal-x
 *   xdbl  (batch, Lseq, K, Cp)      fp32: x_proj output per POSITION and direction (K = 4 / 2 / 1), row =
 *                                   [B (N) | C (N) | dt_r (R) | 0-pad], Cp = sigma_ss2d_padded_cp(N, R)
 *   y     (K, batch, Lseq, D)       fp32: direction k's output stored at the POSITION it belongs
 *                                   to (so CrossMerge is a plain sum over k)
 *   dtw (Kw, D, R), dtb (Kw, D), A (Kw·D, N) [= -exp(A_logs)], Ds (Kw·D); Kw = K, or 2 (modalities) for CROSS
 * ------------------------------------------------------------------------------------------ */
#define SIGMA_DIRS_CROSS4 0 /* K=4: row-major, column-major, and both reversed (vmamba.py:86-88) */
#define SIGMA_DIRS_SEQ2 1   /* K=2: forward and reversed over a flat sequence (vmamba.py:130-131) */
#define SIGMA_DIRS_CROSS 2  /* K=1 per modality, C taken from the other modality (vmamba.py:1530,1536) */

int sigma_ss2d_padded_cp(int N, int R); /* row length of xdbl, or -1 if R > 64 */
size_t sigma_ss2d_scan_workspace_bytes(int kind, int batch, int H, int W, int D, int N);

int sigma_ss2d_scan_fwd(int kind, const float *xc, const float *xdbl, const float *dtw,
                        const float *dtb, const float *A, const float *Ds, float *y,
                        int batch, int H, int W, int D, int N, int R, int Cp,
                        void *workspace, size_t workspace_bytes, void *stream);

/* bf16 inference mode: the same scan with xc and y in bf16 (x_dbl, the parameters, the state and the recurrence fp32; y rounded once
 * on its store).  D % 8 == 0.  Training has its own pair: sigma_ss2d_scan_fwd_save_bf16 / sigma_ss2d_scan_bwd_saved_bf16.        */
int sigma_ss2d_scan_fwd_bf16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                             const float *Ds, void *y, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                             size_t workspace_bytes, void *stream);
/* fp16 inference mode (sigma_b200.fused.fp16_inference): the same with xc and y in fp16 and the launch plan of the bf16 call.
 * Every fp16 store below rounds once to nearest even; a value past ±65504 is stored as ±inf, as torch's .half() does.        */
int sigma_ss2d_scan_fwd_fp16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                             const float *Ds, void *y, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                             size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------
 * f1. Training pair of the fused scan.  `sigma_ss2d_scan_fwd_save` is sigma_ss2d_scan_fwd that also writes what its backward
 * needs: delta (K, batch, Lseq, D) = softplus(dt_proj) at the position it belongs to, and hs (sigma_ss2d_scan_hs_bytes) = the
 * scan state at the start of every 16-position block of each direction's walk (the role of the reference's chunk states `x`,
 * selective_scan_fwd_kernel.cuh:176-190).  `sigma_ss2d_scan_bwd_saved` consumes them (delta and hs are inputs) in one reverse
 * sweep and replaces the autograd of CrossScan (vmamba.py:80-98) + the dt_proj einsum (:199) + SelectiveScan
 * (selective_scan_bwd_kernel.cuh:68-274) + CrossMerge (:100-121) without materialising the (B,4,D,L) copies.
 * kind = SIGMA_DIRS_CROSS4, SIGMA_DIRS_SEQ2 or SIGMA_DIRS_CROSS (batch = 2·images, as the forward; K = 1 walk of ceil(L/16)
 * blocks per image, Kw = 2 weight sets); d_state in {4, 16}; D % 64 == 0 for the backward.  nsplit = 0 lets the library choose
 * the L-segments; otherwise it forces their count (the forward caps it at 32, the backward at 64, both at the tile count of the
 * longest walk), and the two calls may be cut differently.  The backward's inputs are the forward's, delta, hs and
 *   dy      (batch, Lseq, D)      gradient of the MERGED output y = sum_k y_k (CrossMerge is a sum, so every direction sees dy)
 * Outputs (fp32):
 *   dxc     (batch, Lseq, D)      sum over directions of du, accumulated by TMA reduce-add (zeroed inside)
 *   ddelta  (K, batch, Lseq, D)   gradient w.r.t. the PRE-softplus dt_proj output, per direction, at the position it belongs to; the
 *                                 caller finishes d dt_r = ddelta_k · W_dt[k] and dW_dt[k] = ddelta_k^T · dt_r_k with two GEMMs
 *   dxdbl   (batch, Lseq, K, Cp)  dB in columns [0, N), dC in [N, 2N) (zeroed inside; dt_r columns left 0 for the caller); CROSS:
 *                                 image b's dC goes to the C columns of image (b + batch/2) mod batch, whose row supplied C
 *   dA (Kw·D, N), dDs (Kw·D), ddtb (Kw, D)   overwritten; CROSS: rows w·D + d summed over the images of modality w
 * ------------------------------------------------------------------------------------------ */
size_t sigma_ss2d_scan_hs_bytes(int kind, int batch, int H, int W, int D, int N);
size_t sigma_ss2d_scan_bwd_workspace_bytes(int kind, int batch, int H, int W, int D, int N);
int sigma_ss2d_scan_fwd_save(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                             const float *Ds, float *y, float *delta, float *hs, int batch, int H, int W, int D, int N, int R, int Cp,
                             void *workspace, size_t workspace_bytes, int nsplit, void *stream);
int sigma_ss2d_scan_bwd_saved(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A, const float *Ds,
                              const float *dy, const float *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl, float *dA,
                              float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                              size_t workspace_bytes, int nsplit, void *stream);

/* bf16 training mode of the pair above: xc, y, delta and dy are bf16 (16-byte aligned, D % 8 == 0 for the forward, D % 64 == 0 for
 * the backward); x_dbl, hs, the parameters, the state, every accumulator and dxc / ddelta / dxdbl / dA / dDs / ddtb stay fp32
 * (dxc is the fp32 accumulator of the directions' TMA reduce-adds; the caller rounds it once after adding dxdbl · xw).
 * delta = softplus(dt_proj) is rounded to bf16 (nearest even) BEFORE the forward's recurrence uses it, so the backward recomputes
 * exp(delta·A) from exactly the value the forward ran on; y is rounded once on its store.  Same workspace and hs queries, same
 * nsplit convention, same kinds; d_state 4 / 16 (8: SIGMA_EUNSUPPORTED).  No deterministic build. */
int sigma_ss2d_scan_fwd_save_bf16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                  const float *Ds, void *y, void *delta, float *hs, int batch, int H, int W, int D, int N, int R, int Cp,
                                  void *workspace, size_t workspace_bytes, int nsplit, void *stream);
int sigma_ss2d_scan_bwd_saved_bf16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                   const float *Ds, const void *dy, const void *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl,
                                   float *dA, float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                                   size_t workspace_bytes, int nsplit, void *stream);

/* fp16 training mode of the pair (fp16 autocast with a loss scaler such as torch.amp.GradScaler): the _bf16 pair's arguments,
 * validation, workspace / hs queries, kinds and d_state set, with xc, y, delta and dy in fp16.  Every fp16 store rounds once to
 * nearest even and nothing saturates: a value past ±65504 is stored as ±inf, as torch's .half() does, and an inf or NaN in xc or
 * dy reaches the outputs (a loss scaler needs to see it to skip the step).  delta is rounded to fp16 before the forward's
 * recurrence uses it, in the summary pass of an L-segmented walk too; a delta below 2^-14 is stored subnormal and the recurrence
 * runs on that same value, so the backward recomputes exp(delta·A) from exactly what the forward used.  dxc and every other
 * backward output are fp32 (the caller rounds dxc once).  No deterministic build. */
int sigma_ss2d_scan_fwd_save_fp16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                  const float *Ds, void *y, void *delta, float *hs, int batch, int H, int W, int D, int N, int R, int Cp,
                                  void *workspace, size_t workspace_bytes, int nsplit, void *stream);
int sigma_ss2d_scan_bwd_saved_fp16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                   const float *Ds, const void *dy, const void *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl,
                                   float *dA, float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                                   size_t workspace_bytes, int nsplit, void *stream);

/* Deterministic build of the fused backward (after sigma_ss2d_scan_fwd_save): the same outputs, bitwise
 * reproducible for the same inputs, GPU model and L-segment plan.  Each direction's du goes to a slab summed over k into dxc,
 * dB / dC are kept per warp channel tile and dA / dDs / ddtb per (image, L-segment), all in the workspace, then summed in a
 * fixed order; no float atomics and no bulk reduce.  nsplit = 0 lets the library choose the L-segments.  CROSS4 / SEQ2 only: kind
 * CROSS has no deterministic build (SIGMA_EINVAL; the workspace query returns 0) — under the deterministic switch CroMB trains
 * through the op-level _det kernels. */
size_t sigma_ss2d_scan_bwd_det_workspace_bytes(int kind, int batch, int H, int W, int D, int N);
int sigma_ss2d_scan_bwd_saved_det(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                  const float *Ds, const float *dy, const float *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl,
                                  float *dA, float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                                  size_t workspace_bytes, int nsplit, void *stream);

/* ------------------------------------------------------------------------------------------
 * Row-wise / stencil pieces of a5-a11 (channels-last, fp32; D % 4 == 0, 16-byte aligned rows).
 * ------------------------------------------------------------------------------------------ */
/* nn.LayerNorm over the last dim (vmamba.py:1693,724,2173; eps=1e-5): y = (x-mean)/sqrt(var+eps)·w+b */
int sigma_layernorm_fwd(const float *x, const float *w, const float *b, float *y, int64_t rows,
                        int C, float eps, void *stream);
/* bf16 inference mode: the same LayerNorm (fp32 statistics) with y stored as bf16 (8-byte aligned), to feed sigma_linear_bf16. */
int sigma_layernorm_fwd_bf16(const float *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream);
/* fp16 inference mode: the same with y stored as fp16, to feed sigma_linear_fp16. */
int sigma_layernorm_fwd_fp16(const float *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream);
/* bf16 training mode: x and y both bf16 (8-byte aligned rows), fp32 statistics, w and b. */
int sigma_layernorm_fwd_bf16io(const void *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream);
/* fp16 training mode: x and y both fp16 (8-byte aligned rows), fp32 statistics, w and b; y rounds once, past ±65504 to ±inf. */
int sigma_layernorm_fwd_fp16io(const void *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream);

/* Backward of sigma_layernorm_fwd (training path; the reference's autograd of nn.LayerNorm): dx (rows, C); dw (C) = sum over rows
 * of dy·xhat, db (C) = sum over rows of dy — both zeroed inside, then accumulated.  mean / rstd are recomputed from x.
 * C/4 must be one of {8, 16, 24, 32, 48, 64, 96, 128, 192, 256, 384} (every Sigma width up to 1536); else SIGMA_EUNSUPPORTED. */
int sigma_layernorm_bwd(const float *x, const float *dy, const float *w, float *dx, float *dw, float *db, int64_t rows, int C,
                        float eps, void *stream);
/* The same with bf16 x, dy and dx (8-byte aligned rows; the backward of sigma_layernorm_fwd_bf16io): statistics, dw and db fp32.
 * No deterministic build. */
int sigma_layernorm_bwd_bf16(const void *x, const void *dy, const float *w, void *dx, float *dw, float *db, int64_t rows, int C,
                             float eps, void *stream);
/* The same with fp16 x, dy and dx (the backward of sigma_layernorm_fwd_fp16io): dx rounds once, past ±65504 to ±inf, and an inf or
 * NaN in x or dy reaches dx, dw and db.  No deterministic build. */
int sigma_layernorm_bwd_fp16(const void *x, const void *dy, const float *w, void *dx, float *dw, float *db, int64_t rows, int C,
                             float eps, void *stream);
/* Deterministic build: dw / db kept per warp in the (16-byte aligned) workspace and summed in warp order; no float atomics. */
size_t sigma_layernorm_bwd_det_workspace_bytes(int64_t rows, int C);
int sigma_layernorm_bwd_det(const float *x, const float *dy, const float *w, float *dx, float *dw, float *db, int64_t rows, int C,
                            float eps, void *workspace, size_t workspace_bytes, void *stream);

/* Backward of F.interpolate(mode="bilinear", align_corners=False), fp32, gather form (deterministic: every input element sums
 * the output elements that tap it in a fixed order).  dy (batch, C, Hout, Wout) -> dx (batch, C, Hin, Win), NCHW, or with
 * channels_last = 1 (batch, Hout, Wout, C) -> (batch, Hin, Win, C).  ratio_h / ratio_w are torch's source-index scales rounded
 * to fp32: 1/scale_factor when the forward was given one, Hin/Hout (Win/Wout) when it was given a size. */
int sigma_upsample_bilinear_bwd(const float *dy, float *dx, int batch, int C, int Hin, int Win, int Hout, int Wout, float ratio_h,
                                float ratio_w, int channels_last, void *stream);

/* PatchMerging2D front half (vmamba.py:619-633): y[b,i,j,:] = LayerNorm(cat(x[b,2i,2j], x[b,2i+1,2j], x[b,2i,2j+1],
 * x[b,2i+1,2j+1])) over 4C channels, zero rows beyond an odd H / W (F.pad).  x (batch,H,W,C) -> y (batch,⌈H/2⌉,⌈W/2⌉,4C);
 * the gather is index math inside the LayerNorm kernel (no concatenated tensor).  4C must be 32·k·{2,3,4,6,8,12,16}-shaped
 * (every Sigma width is).                                                                    */
int sigma_patch_merge_norm_fwd(const float *x, const float *w, const float *b, float *y, int batch, int H, int W,
                               int C, float eps, void *stream);
/* bf16 inference mode: the same gather + LayerNorm with y stored as bf16 (8-byte aligned).                                      */
int sigma_patch_merge_norm_fwd_bf16(const float *x, const float *w, const float *b, void *y, int batch, int H, int W, int C,
                                    float eps, void *stream);
/* fp16 inference mode: the same with y stored as fp16. */
int sigma_patch_merge_norm_fwd_fp16(const float *x, const float *w, const float *b, void *y, int batch, int H, int W, int C,
                                    float eps, void *stream);

/* PatchExpand back half (MambaDecoder.py:24-30): x is the expand Linear's output (batch,H,W,2,2,C) ("b h w (p1 p2 c)"),
 * y[b,2h+p1,2w+p2,:] = LayerNorm(x[b,h,w,p1,p2,:]); y (batch,2H,2W,C).  The pixel shuffle is the store address.   */
int sigma_pixel_shuffle_norm_fwd(const float *x, const float *w, const float *b, float *y, int batch, int H, int W,
                                 int C, float eps, void *stream);

/* depthwise 3x3 conv (pad 1) + bias + SiLU, channels-last (vmamba.py:683-692,1072).
 * x: position rows x_row_stride floats apart, images x_batch_stride apart (so the x half of
 * in_proj's (.., 2D) output is read in place); w is the nn.Conv2d weight (D,1,3,3) contiguous;
 * y: (H·W, D) rows per image, images y_batch_stride floats apart.                         */
int sigma_dwconv3x3_silu_fwd(const float *x, int64_t x_row_stride, int64_t x_batch_stride,
                             const float *w, const float *bias, float *y, int64_t y_batch_stride,
                             int batch, int H, int W, int D, void *stream);
/* bf16 inference mode: the same depthwise conv + SiLU with x and y bf16 (fp32 weights, bias and accumulation).  x 16-byte aligned,
 * x strides multiples of 8 elements (TMA); y 8-byte aligned, y_batch_stride % 4 == 0.                                          */
int sigma_dwconv3x3_silu_fwd_bf16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  void *y, int64_t y_batch_stride, int batch, int H, int W, int D, void *stream);
/* fp16 inference mode: the same with x and y fp16. */
int sigma_dwconv3x3_silu_fwd_fp16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  void *y, int64_t y_batch_stride, int batch, int H, int W, int D, void *stream);

/* Backward of sigma_dwconv3x3_silu_fwd (training: the autograd of nn.Conv2d(D, D, 3, padding=1, groups=D) + SiLU).  With
 * pre = conv(x) + b recomputed from x and s = sigmoid(pre):
 *   g = dy·s·(1 + pre·(1 − s)),  dx = the transposed stencil of g (flipped taps),
 *   dw[c, tap] = Σ over images and pixels of g·(x at the tap's shift),  dbias = Σ g.
 * x as in the forward (position rows x_row_stride elements apart, images x_batch_stride apart); dy and dx (H·W, D) rows per image,
 * images dy_batch_stride / dx_batch_stride elements apart; dw (D,1,3,3) and dbias (D) fp32, overwritten.  bias and dbias may be
 * NULL together.  Deterministic by construction (no float atomics): each CTA sums its tiles in a fixed order into one partial row
 * of the caller's workspace (sigma_dwconv3x3_silu_bwd_workspace_bytes, 16-byte aligned), and the rows are added in order, so the
 * same inputs give the same bits with or without a deterministic mode.  D % 4 == 0; x, dy, dx 16-byte aligned, strides multiples
 * of 4 elements.                                                                                                              */
size_t sigma_dwconv3x3_silu_bwd_workspace_bytes(int batch, int H, int W, int D);
int sigma_dwconv3x3_silu_bwd(const float *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                             const float *dy, int64_t dy_batch_stride, float *dx, int64_t dx_batch_stride, float *dw, float *dbias,
                             int batch, int H, int W, int D, void *workspace, size_t workspace_bytes, void *stream);
/* bf16 / fp16 training: the same with x, dy and dx 16-bit (D % 8 == 0, strides multiples of 8 elements).  g, every sum, dw and
 * dbias are fp32; dx rounds once (fp16: past ±65504 to ±inf).  The same workspace.                                             */
int sigma_dwconv3x3_silu_bwd_bf16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  const void *dy, int64_t dy_batch_stride, void *dx, int64_t dx_batch_stride, float *dw, float *dbias,
                                  int batch, int H, int W, int D, void *workspace, size_t workspace_bytes, void *stream);
int sigma_dwconv3x3_silu_bwd_fp16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  const void *dy, int64_t dy_batch_stride, void *dx, int64_t dx_batch_stride, float *dw, float *dbias,
                                  int batch, int H, int W, int D, void *workspace, size_t workspace_bytes, void *stream);

/* CrossMerge sum + out_norm LayerNorm + gates (vmamba.py:217-224,1077; ConMB: 423-428,1280-1281):
 *   out[r,:] = (LN(Σ_k y[k][r,:])·gamma+beta) · (z ? SiLU(z[r,:]) : 1) · (gate ? gate[r / rows_per_batch, :] : 1)
 * Row r = (b, i) with b = r / rows_per_batch: input row at y + k·k_stride + b·in_batch_stride + i·D,
 * output row at out + b·out_batch_stride + i·out_row_stride, z row at z + r·z_row_stride.     */
int sigma_merge_norm_gate_fwd(const float *y, int K, int64_t k_stride, int64_t in_batch_stride,
                              const float *gamma, const float *beta, const float *z,
                              int64_t z_row_stride, const float *gate, float *out,
                              int64_t out_batch_stride, int64_t out_row_stride, int64_t rows,
                              int64_t rows_per_batch, int D, float eps, void *stream);
/* bf16 inference mode: the same merge + LayerNorm + gates with y, z and out bf16 (8-byte aligned); gamma, beta, gate and the
 * statistics fp32.  Strides count elements.                                                                                   */
int sigma_merge_norm_gate_fwd_bf16(const void *y, int K, int64_t k_stride, int64_t in_batch_stride, const float *gamma,
                                   const float *beta, const void *z, int64_t z_row_stride, const float *gate, void *out,
                                   int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch,
                                   int D, float eps, void *stream);
/* fp16 inference mode: the same with y, z and out fp16. */
int sigma_merge_norm_gate_fwd_fp16(const void *y, int K, int64_t k_stride, int64_t in_batch_stride, const float *gamma,
                                   const float *beta, const void *z, int64_t z_row_stride, const float *gate, void *out,
                                   int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch,
                                   int D, float eps, void *stream);

/* UpsampleExpand tail (MambaDecoder.py:47-49): y = LayerNorm(bilinear x2 (align_corners=False) of x); x (batch,H,W,C),
 * y (batch,2H,2W,C).  One pass: the upsampled tensor is never materialised un-normalised.
 * w == b == NULL: plain bilinear x2 without the LayerNorm (FinalUpsample_X4's first interpolate, MambaDecoder.py:92). */
int sigma_upsample2x_norm_fwd(const float *x, const float *w, const float *b, float *y, int batch, int H, int W, int C,
                              float eps, void *stream);

/* FinalUpsample_X4 tail + classifier (MambaDecoder.py:95-96, 276-279): logits = Conv1x1(LayerNorm(bilinear x2 (x))).
 * x (batch,H,W,C); wcls (num_classes, C) = the 1x1 conv weight; logits (batch, num_classes, 2H, 2W) NCHW.   */
int sigma_upsample2x_norm_head_fwd(const float *x, const float *w, const float *b, const float *wcls, int num_classes,
                                   float *logits, int batch, int H, int W, int C, float eps, void *stream);

/* ChannelAttention pooling (vmamba.py:1738-1739): per-slice partial sums and maxima over the L positions of each image,
 * x (batch, L, C) channels-last -> partial (batch, nslice, 2, C) [0]=sum [1]=max (the caller finishes the tiny reduction). */
int sigma_pool_avgmax_partial_fwd(const float *x, float *partial, int batch, int64_t L, int C, int nslice, void *stream);

/* out[r,:] = a[r,:]·sa[r / rows_per_batch, :] + b[r,:]·sb[:]   (a, sa nullable: out = b·sb).  CVSSDecoderBlock residuals
 * (vmamba.py:1801,1803) with the channel-attention scaling (vmamba.py:1741) folded in.                      */
int sigma_scale_add_fwd(const float *a, const float *sa, const float *b, const float *sb, float *out, int64_t rows,
                        int64_t rows_per_batch, int C, void *stream);

/* ------------------------------------------------------------------------------------------
 * Dense projections (in_proj / x_proj / out_proj / PatchMerging / PatchExpand / decoder linears,
 * vmamba.py:679,725,616,195; MambaDecoder.py:17,39,82-83): hand-written Hopper wgmma TF32 GEMM,
 * fp32 storage, fp32 accumulate in registers, TMA-fed, fused epilogue:
 *     C[M,N] = A[M,K]·W[N,K]^T (+ bias[N]) (+ residual[M,N] (· rscale[N]))
 * A rows lda floats apart, W (N,K) contiguous, C rows ldc apart, residual rows ldr apart; K, lda, ldc, ldr % 4 == 0.
 * rscale is the per-channel residual scale of CVSSDecoderBlock (vmamba.py:1801); bias/residual/rscale nullable.
 * ------------------------------------------------------------------------------------------ */
int sigma_linear_tf32(const float *A, int64_t lda, const float *W, const float *bias, const float *residual, int64_t ldr,
                      const float *rscale, float *C, int64_t ldc, int64_t M, int N, int K, void *stream);

/* The same GEMM with fp32-GRADE products on the TF32 tensor pipe ("tf32x3": A·W = A_hi·W_hi + A_lo·W_hi + A_hi·W_lo, x_hi = x with
 * the low 13 mantissa bits cleared; three wgmma MMAs per k-step, activations split in registers inside the kernel): what
 * torch's nn.Linear computes with torch.backends.cuda.matmul.allow_tf32 = False, to ~1e-6 relative.  The weights arrive
 * pre-split (W_hi, W_lo each (N, K) contiguous): split them once with sigma_split_tf32_fwd.                                  */
int sigma_linear_tf32x3(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias, const float *residual,
                        int64_t ldr, const float *rscale, float *C, int64_t ldc, int64_t M, int N, int K, void *stream);
int sigma_split_tf32_fwd(const float *x, float *hi, float *lo, int64_t n, void *stream);

/* bf16 inference mode: the same GEMM on bf16 operands (`wgmma ... k16.f32.bf16.bf16`, one MMA per 16-wide k-step, fp32 accumulate):
 * A (M, K) bf16 rows lda elements apart, W (N, K) bf16 contiguous; C rows ldc elements apart, stored as fp32 (c_dtype = SIGMA_F32)
 * or bf16 (SIGMA_BF16, rounded once); bias / residual / rscale fp32.  K, lda % 8 == 0; N, ldc, ldr % 4 == 0; 16-byte aligned.   */
int sigma_linear_bf16(const void *A, int64_t lda, const void *W, const float *bias, const float *residual, int64_t ldr,
                      const float *rscale, void *C, int64_t ldc, int c_dtype, int64_t M, int N, int K, void *stream);
/* fp16 inference mode: the same GEMM on fp16 operands (`wgmma ... k16.f32.f16.f16`), the same tile widths and launch plan; C fp32
 * (c_dtype = SIGMA_F32) or fp16 (SIGMA_F16, rounded once: past ±65504 it is ±inf).                                             */
int sigma_linear_fp16(const void *A, int64_t lda, const void *W, const float *bias, const float *residual, int64_t ldr,
                      const float *rscale, void *C, int64_t ldc, int c_dtype, int64_t M, int N, int K, void *stream);

/* ------------------------------------------------------------------------------------------
 * FP8 inference mode (sigma_b200.fused.fp8_inference): e4m3 operands with fp32 scales.
 * Quantizing a row x[0..C) (an activation row, or a weight's output channel) — every step one IEEE fp32 operation, round to
 * nearest even:
 *     amax = max_i |x_i|                     (fp32 values as the producer computed them, before any bf16 rounding)
 *     amax == 0:  s = 1,  q_i = 0
 *     otherwise:  inv = min(448 / amax, FLT_MAX),  s = amax / 448,
 *                 q_i = cvt.rn.satfinite.e4m3(x_i · inv)   (round to nearest even, subnormals kept, |q| clamped to 448)
 * so that x_i ≈ q_i · s.  The GEMM multiplies its fp32 accumulator by s_a[row] · s_w[col] (in that order) before the bias and
 * residual epilogue.
 * ------------------------------------------------------------------------------------------ */
/* C[M,N] = (A[M,K]·Wq[N,K]^T)·sa[m]·sw[n] (+ bias[N]) (+ residual[M,N] (· rscale[N])) on the e4m3 tensor cores (`wgmma ...
 * k32.f32.e4m3.e4m3`): A (M, K) e4m3 rows lda bytes apart, Wq (N, K) e4m3 contiguous, sa (M) and sw (N) fp32; each 128-wide
 * k-block accumulates separately and is added to fp32 accumulators in registers.  C rows ldc elements apart, fp32 (c_dtype =
 * SIGMA_F32) or bf16 (SIGMA_BF16); bias / residual / rscale fp32.  K, lda % 16 == 0; N, ldc, ldr % 4 == 0; A, Wq, C, bias,
 * residual, rscale 16-byte aligned.                                                                                              */
int sigma_linear_fp8(const void *A, int64_t lda, const float *sa, const void *Wq, const float *sw, const float *bias, const float *residual,
                     int64_t ldr, const float *rscale, void *C, int64_t ldc, int c_dtype, int64_t M, int N, int K, void *stream);
/* Row quantizer (the formula above): x (rows, C) fp32 (x_dtype = SIGMA_F32, 16-byte aligned) or bf16 (SIGMA_BF16, 8-byte aligned)
 * rows ldx elements apart -> q (rows, C) e4m3 rows ldq bytes apart (4-byte aligned) and scale (rows) fp32.  C, ldx, ldq % 4 == 0.
 * Weights are quantized per output channel with it; so are activations that no row-wise producer below emits.               */
int sigma_quantize_e4m3_rows(const void *x, int x_dtype, int64_t ldx, void *q, int64_t ldq, float *scale, int64_t rows, int C, void *stream);
/* The producers of the FP8 mode that hold a whole row in registers, with a quantizing output: the same arithmetic as
 * sigma_layernorm_fwd, sigma_patch_merge_norm_fwd and sigma_merge_norm_gate_fwd_bf16 (K = 1 or 4 there), the fp32 result quantized
 * by the formula above into q (e4m3, the output layout of the plain call, in bytes; 4-byte aligned) and scale[r] for row r (the
 * row index of the call: b·rows_per_batch + i for the merge).                                                                  */
int sigma_layernorm_fwd_fp8(const float *x, const float *w, const float *b, void *q, float *scale, int64_t rows, int C, float eps,
                            void *stream);
int sigma_patch_merge_norm_fwd_fp8(const float *x, const float *w, const float *b, void *q, float *scale, int batch, int H, int W, int C,
                                   float eps, void *stream);
int sigma_merge_norm_gate_fwd_fp8(const void *y, int K, int64_t k_stride, int64_t in_batch_stride, const float *gamma,
                                  const float *beta, const void *z, int64_t z_row_stride, const float *gate, void *q, float *scale,
                                  int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch,
                                  int D, float eps, void *stream);

/* Dense 3x3 convolution (pad 1, stride 1) of the ChannelAttentionBlock (vmamba.py:1749-1752), channels-last, as an implicit GEMM on
 * the same wgmma kernel: y (batch, H, W, Cout) = conv(x (batch, H, W, Cin), w9) + bias, act = 1 applies the exact (erf) GELU of
 * nn.GELU() in the epilogue.  w9 = the nn.Conv2d weight (Cout, Cin, 3, 3) re-ordered to (3·3, Cout, Cin); every tap's input patch
 * is one shifted 4-D TMA box whose out-of-bounds fill is the zero padding.  w9_lo == NULL: one TF32 MMA per k-step; otherwise
 * tf32x3 with (w9, w9_lo) = sigma_split_tf32_fwd of the re-ordered weight.  Cin, Cout % 4 == 0.                              */
int sigma_conv3x3_tf32(const float *x, const float *w9, const float *w9_lo, const float *bias, int act, float *y, int batch, int H, int W,
                       int Cin, int Cout, void *stream);

/* Training of conv3x3 + GELU (the ChannelAttentionBlock's first conv and its activation; ops.CabConvFn).  Same layouts, precision
 * rule (w9_lo) and checks as sigma_conv3x3_tf32.  Forward that keeps the pre-activation: pre = conv(x, w9) + bias and
 * y = GELU(pre) (exact, erf), both (batch, H, W, Cout).  bias may be NULL.                                                   */
int sigma_conv3x3_gelu_save_tf32(const float *x, const float *w9, const float *w9_lo, const float *bias, float *y, float *pre, int batch,
                                 int H, int W, int Cin, int Cout, void *stream);
/* Data gradient of a 3x3 conv (pad 1) with Cin inputs and Cout outputs: dx (batch, H, W, Cin) = the 3x3 conv of dy (batch, H, W, Cout)
 * with w9t (3·3, Cin, Cout), the weight flipped in the taps and transposed: w9t[tap][ci][co] = w[co][ci][8 − tap] of the nn.Conv2d
 * weight w (Cout, Cin, 3, 3) (w9t_lo: its tf32x3 split, or NULL for TF32).  gelu_pre != NULL (batch, H, W, Cin): dx is multiplied
 * by GELU'(gelu_pre) = Φ(u) + u·φ(u), the gradient at the pre-activation of a GELU that fed the conv.  Cin, Cout % 4 == 0.     */
int sigma_conv3x3_dgrad_tf32(const float *dy, const float *w9t, const float *w9t_lo, const float *gelu_pre, float *dx, int batch, int H,
                             int W, int Cin, int Cout, void *stream);
/* Weight gradient of the same conv: dw (Cout, Cin, 3, 3) = Σ over pixels of dy[p, co]·x[p + s(tap), ci] (nn.Conv2d's layout) and
 * dbias (Cout) = Σ dy (NULL: not computed); x (batch, H, W, Cin) or, gelu_x = 1, the pre-activation whose GELU was the conv's input.
 * x3 = 0: one TF32 MMA per k-step; 1: tf32x3 (fp32 grade).  Deterministic by construction: each CTA sums a fixed pixel range into one
 * partial row of the caller's workspace (sigma_conv3x3_wgrad_workspace_bytes, 16-byte aligned), and the rows are added in order, so
 * the same inputs give the same bits with or without a deterministic mode.  Cin, Cout % 4 == 0; x, dy 16-byte aligned.            */
size_t sigma_conv3x3_wgrad_workspace_bytes(int batch, int H, int W, int Cin, int Cout);
int sigma_conv3x3_wgrad_tf32(const float *x, int gelu_x, const float *dy, float *dw, float *dbias, int batch, int H, int W, int Cin,
                             int Cout, int x3, void *workspace, size_t workspace_bytes, void *stream);
/* Launch plan of sigma_conv3x3_wgrad_tf32, host only (no CUDA call): out4_host = {output channels per tile, output tiles, partial
 * rows (pixel ranges), CTAs}.  A function of the shape alone.                                                                  */
int sigma_test_conv3x3_wgrad_plan(int batch, int H, int W, int Cin, int Cout, int64_t *out4_host);

/* The four calls above on pitched rows, for channel counts that are not multiples of 4 (the CAB convs of Sigma-base, whose C/3 is
 * 42 / 85 / 170; ops.CabConvPitchedFn, fused.cvss_decoder_block).  Each activation and weight is given with its row pitch in
 * elements: a multiple of 4, at least its channel count.  Channels between the count and the pitch are pad: never read into a kept
 * output (the conv's tensor maps end at the count, so TMA fills zeros past it) and never written.  Weights are the layouts above
 * with rows at the pitch: w9 (9·Cout rows of Cin at w9_pitch), w9t (9·Cin rows of Cout at w9t_pitch), w9_lo / w9t_lo (or NULL) at
 * the same pitch.  dw and dbias keep nn.Conv2d's unpadded layout, and the weight gradient's workspace is
 * sigma_conv3x3_wgrad_workspace_bytes (the same plan).  x, y, pre (at y_pitch), dy, dx and gelu_pre (at dx_pitch) 16-byte
 * aligned.  With every pitch equal to its count (a multiple of 4), each call computes what its unpitched twin does.           */
int sigma_conv3x3_pitched_tf32(const float *x, int x_pitch, const float *w9, int w9_pitch, const float *w9_lo, const float *bias, int act,
                               float *y, int y_pitch, int batch, int H, int W, int Cin, int Cout, void *stream);
int sigma_conv3x3_gelu_save_pitched_tf32(const float *x, int x_pitch, const float *w9, int w9_pitch, const float *w9_lo,
                                         const float *bias, float *y, float *pre, int y_pitch, int batch, int H, int W, int Cin, int Cout,
                                         void *stream);
int sigma_conv3x3_dgrad_pitched_tf32(const float *dy, int dy_pitch, const float *w9t, int w9t_pitch, const float *w9t_lo,
                                     const float *gelu_pre, float *dx, int dx_pitch, int batch, int H, int W, int Cin, int Cout,
                                     void *stream);
int sigma_conv3x3_wgrad_pitched_tf32(const float *x, int x_pitch, int gelu_x, const float *dy, int dy_pitch, float *dw, float *dbias,
                                     int batch, int H, int W, int Cin, int Cout, int x3, void *workspace, size_t workspace_bytes,
                                     void *stream);

/* Launch plan of the two calls above, host only (no CUDA call, works without a GPU): what sigma_linear_tf32{,x3} (conv_B = 0; M rows,
 * N outputs, K inputs) or sigma_conv3x3_tf32 (conv_B > 0: input (conv_B, conv_H, conv_W, K), N = Cout; M unused) would launch under
 * the current environment.  out6_host = {tile width, ring stages, persistent grid, output tiles, dynamic shared memory bytes, CTAs
 * per SM}.  The environment variable SIGMA_GEMM_BN=<w> forces the tile width of both calls (a multiple of 32 in [32, 256], read
 * per call; any other value makes the calls and this query return SIGMA_EINVAL).  For tests and tuning.
 * x3 selects the instance: 0 = tf32, 1 = tf32x3 with register-stored output tiles (the conv and
 * sigma_test_linear_tf32x3_regs), 2 = sigma_linear_bf16, 4 = sigma_linear_fp8, 5 = tf32x3 with TMA-stored output tiles
 * (sigma_linear_tf32x3), 7 = sigma_linear_fp16 (the plan of 2); conv_B must be 0 for 2, 4, 5 and 7; the e4m3 tiles are 32 or 64
 * wide, and forcing a wider one is SIGMA_EINVAL; other values (3 and 6 included) are SIGMA_EINVAL.                            */
int sigma_test_gemm_plan(int64_t M, int N, int K, int x3, int conv_B, int conv_H, int conv_W, int64_t *out6_host);
/* sigma_linear_tf32x3 (same arguments and checks) with the output tiles stored from registers instead of through shared memory
 * and TMA: the same products and epilogue operations, so the same bits.  For tests.                                          */
int sigma_test_linear_tf32x3_regs(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias,
                                  const float *residual, int64_t ldr, const float *rscale, float *C, int64_t ldc, int64_t M, int N,
                                  int K, void *stream);

/* L-segment plan of the fused scan backward, host only (no CUDA call, works without a GPU): what sigma_ss2d_scan_bwd_saved with
 * that nsplit (0: the library's choice) would launch for kind CROSS4 / SEQ2 / CROSS (even
 * batch) at (batch, H, W, D, N).  out4_host = {segments, 16-position tiles per segment, tiles of the longest direction's walk, tiles of the shortest}.  The
 * directions share the tiles per segment, so a walk shorter than the longest can end in empty segments.  The plan does not depend
 * on the element type: sigma_ss2d_scan_bwd_saved_bf16 / _fp16 launch the same segments.  For tests and tuning. */
int sigma_test_ss2d_bwd_plan(int kind, int batch, int H, int W, int D, int N, int nsplit, int64_t *out4_host);

/* Launch plan of the fused scan forward, host only (no CUDA call, works without a GPU): what sigma_ss2d_scan_fwd (force_split = 0),
 * sigma_ss2d_scan_fwd_split (force_split > 0) or, with bf16 = 1, sigma_ss2d_scan_fwd_bf16 (bf16 = 2: sigma_ss2d_scan_fwd_save_bf16
 * with nsplit = force_split; d_state 8 is SIGMA_EUNSUPPORTED there; bf16 = 3: sigma_ss2d_scan_fwd_fp16; bf16 = 4:
 * sigma_ss2d_scan_fwd_save_fp16, whose plan is that of bf16 = 2 and which refuses d_state 8 as well) would launch for any kind at (batch, H,
 * W, D, N, R) given a workspace of workspace_bytes (0: none), under the current environment (SIGMA_SCAN_WARPS, SIGMA_SCAN_NST,
 * SIGMA_SCAN_CTAS, SIGMA_SCAN_SPLIT_RULE).  out8_host = {segments, LT-position tiles per segment, tiles of the longest direction's
 * walk, tiles of the shortest, warps per CTA, TMA ring depth, register budget (the CTAs per SM the kernel build assumes: 3 or 4),
 * dynamic shared-memory bytes per CTA}.  Returns what the launch would: SIGMA_EWORKSPACE for force_split > 1 without a large
 * enough workspace.  For tests and tuning.                                                                                     */
int sigma_test_ss2d_fwd_plan(int kind, int batch, int H, int W, int D, int N, int R, int bf16, int force_split, size_t workspace_bytes,
                             int64_t *out8_host);

/* sigma_scan_fwd with a forced number of L-segments (nsplit = 0: the library's choice; more than 64 is capped at 64), any dtype
 * and route.  Without a workspace large enough for the carries the scan runs unsplit.  For tests and tuning.                    */
int sigma_scan_fwd_split(const void *u, const void *delta, const float *A, const void *B, const void *C,
                         const float *D, const float *delta_bias, void *out, float *x,
                         int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                         int delta_softplus, const sigma_scan_strides *strides,
                         void *workspace, size_t workspace_bytes, int nsplit, void *stream);

/* Launch plan of the op-level selective scan, host only (no CUDA call, works without a GPU): what sweep 0 = sigma_scan_fwd{,_split},
 * 1 = sigma_scan_bwd{,_split}, 2 = sigma_scan_bwd_det would launch at (batch, dim, seqlen, dstate, ngroups, dtype) with nsplit
 * forced L-segments (0: the library's choice) and workspace_bytes of workspace, for contiguous 16-byte aligned operands, under
 * the current environment (SIGMA_OP_GENERIC, SIGMA_OP_NST).  out8_host = {route (0 TMA-staged, 1 TMA-staged on fp32 copies of
 * 16-bit operands, 2 generic), segments, position tiles per segment, position tiles, channels per CTA, ring stages, and for the
 * backward the segments and tiles per segment of its state sweep (0 for the forward)}.  The generic backward runs one segment.
 * Returns what the launch would: SIGMA_EWORKSPACE for a backward without its workspace.  For tests and tuning.                  */
int sigma_test_scan_plan(int sweep, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype, int nsplit,
                         size_t workspace_bytes, int64_t *out8_host);

/* ------------------------------------------------------------------------------------------
 * Test hooks: the scans with a forced number of L-segments, and the launch heuristics alone.  For tests and tuning.
 * ------------------------------------------------------------------------------------------ */
/* sigma_scan_bwd with a forced number of L-segments (nsplit = 0: the library's choice; more than 64 is capped at 64).  The generic
 * backward runs one segment.                                                                                                   */
int sigma_scan_bwd_split(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                         const float *delta_bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                         float *dD, float *ddelta_bias, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                         int delta_softplus, void *workspace, size_t workspace_bytes, int nsplit, void *stream);
/* sigma_ss2d_scan_fwd with a forced number of L-segments (nsplit = 0: the library's choice; capped at 32 and at the tile count of
 * the longest walk).  nsplit > 1 without a large enough workspace is SIGMA_EWORKSPACE.                                         */
int sigma_ss2d_scan_fwd_split(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                              const float *Ds, float *y, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                              size_t workspace_bytes, int nsplit, void *stream);
/* Host only (no CUDA call, works without a GPU): the L-segment count the fused scan forward picks for a grid of `ctas` CTAs of
 * warps_per_cta warps walking ntiles tiles at d_state N, and the GEMM tile width for N output columns and m_tiles 128-row tiles. */
int sigma_test_pick_segments(int64_t ctas, int warps_per_cta, int ntiles, int N);
int sigma_test_pick_bn(int N, int64_t m_tiles);

/* ------------------------------------------------------------------------------------------
 * SURVEY.md §8(f) rank 2, first piece: the evaluator's per-batch metric on the device (eval.py:22-29,
 * utils/metric.py:8-15).  pred = argmax over classes of logits (batch, classes, H, W) — the index numpy.argmax
 * returns for exp(score) (evaluator.py:520,449); for labels in [0, classes): hist[label·classes + pred] += 1,
 * counts[0] (labeled) += 1, counts[1] (correct) += (pred == label).  hist (classes²) and counts (2) are uint64
 * ACCUMULATORS in device memory (zero them once per evaluation); labels (batch, H, W) are uint8 / int32 / int64
 * (label_bytes = 1 / 4 / 8), anything outside [0, classes) — e.g. 255 — is ignored; pred (batch·H·W uint8) may be NULL.
 * num_classes <= 238 (the per-CTA histogram lives in shared memory).
 * ------------------------------------------------------------------------------------------ */
int sigma_argmax_hist_fwd(const float *logits, const void *labels, int label_bytes, uint64_t *hist,
                          uint64_t *counts, uint8_t *pred, int batch, int num_classes, int64_t HW,
                          void *stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY.md §8(f) ranks 2 and 3: the callers either side of the hot path, on the device.
 *
 * sigma_image_pre_fwd — the pre-processing of ONE image into one (3, OH, OW) float32 network input (and optionally its
 * (OH, OW) int64 label map): replaces, in one kernel, TrainPre.__call__ (dataloader/dataloader.py:26-50: random_mirror,
 * random_scale = cv2.resize INTER_LINEAR / INTER_NEAREST, normalize, random_crop_pad_to_shape) and the evaluator's
 * process_image_rgbX (engine/evaluator.py:523-558: normalize + pad_image_to_shape) incl. the multi-scale cv2.resize of
 * sliding_eval_rgbX (:439-444) and the horizontal flip of the padded input (:512-515).  The random choices are made by the
 * caller and passed in.  src (H0, W0, 3) uint8 HWC; labels (H0, W0) uint8 or NULL.
 *   scaled image = cv2.resize(src [flipped horizontally first if mirror_src], (SW, SH), INTER_LINEAR), 8-bit fixed-point
 *                  arithmetic of OpenCV's generic path (scale_y / scale_x = source pixels per scaled pixel: 1/fy, 1/fx, or
 *                  H0/SH, W0/SW); SH == H0 and SW == W0: no resize
 *   out(c, oy, ox) = ((scaled(oy + off_y, ox + off_x, c) / 255) - mean[c]) / std[c]  (double, utils/transforms.py:182-187),
 *                    0 outside the scaled image — or outside the rectangle clip4_host = {y0, x0, h, w} of it when given (a sliding
 *                    window, evaluator.py:478-482) —; label_out = label_pad there (255 in TrainPre); mirror_out flips the OUTPUT.
 * ------------------------------------------------------------------------------------------ */
int sigma_image_pre_fwd(const uint8_t *src, const uint8_t *labels, float *out, int64_t *labels_out, int H0, int W0, int SH, int SW,
                        double scale_y, double scale_x, int OH, int OW, int off_y, int off_x, int mirror_src, int mirror_out,
                        int label_pad, const int *clip4_host, const double *mean3_host, const double *std3_host, void *stream);

/* evaluator.py:505-520 and 481-488: acc[c, ay + y, ax + x] += exp(logits[c, m_top + y, m_left + x] (+ logits_flip[c, m_top + y,
 * TW - 1 - (m_left + x)])) for y < vh, x < vw.  logits (ncls, TH, TW) = one image of the model's NCHW output; logits_flip
 * (nullable) = the output for the horizontally flipped input; acc (ncls, AH, AW) float32 = the scale's score map.         */
int sigma_eval_exp_accumulate_fwd(const float *logits, const float *logits_flip, float *acc, int ncls, int TH, int TW, int m_top,
                                  int m_left, int vh, int vw, int AH, int AW, int ay, int ax, void *stream);

/* evaluator.py:497-499 and 447-448: out (H0, W0, ncls) float64 += cv2.resize(acc[:, m_top : m_top + SH, m_left : m_left + SW]
 * as HWC float32, (W0, H0), INTER_LINEAR) (cv2's float path; identity when SH == H0 and SW == W0).                        */
int sigma_eval_resize_add_fwd(const float *acc, int ncls, int AH, int AW, int m_top, int m_left, int SH, int SW, double *out,
                              int H0, int W0, void *stream);

/* evaluator.py:451 + eval.py:28 + utils/metric.py:8-15: pred = argmax over classes of score (HW, ncls) float64 (first maximum,
 * numpy.argmax); labels (HW) uint8 nullable: hist[label·ncls + pred] += 1, counts[0] (labeled) += 1, counts[1] (correct)
 * += (pred == label) for label < ncls.  hist / counts are uint64 accumulators.                                            */
int sigma_eval_argmax_hist_fwd(const double *score, const uint8_t *labels, uint8_t *pred, uint64_t *hist, uint64_t *counts,
                               int num_classes, int64_t HW, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SIGMA_B200_H_ */
