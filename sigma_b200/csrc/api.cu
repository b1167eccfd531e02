// C-ABI entry points (include/sigma_b200.h): argument checking, dtype staging, error strings.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include <atomic>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"

namespace sigma {

static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

// SIGMA_OP_GENERIC=1 forces the generic kernels (A/B timing, tests of the fallback on TMA-eligible shapes)
static bool force_generic() {
  const char *e = getenv("SIGMA_OP_GENERIC");
  return e && atoi(e) > 0;
}

// ---- 16-bit tensors whose rows are not 16-byte aligned (L % 8 != 0, e.g. the 15 x 20 stage) cannot be TMA boxes.  When the
// fp32 image of the call IS eligible (L % 4 == 0), it is cheaper to widen the operands into scratch, run the TMA-staged fp32
// kernels and narrow the results than to take the generic kernels (measured: 0.2-0.6x of the reference kernel there). ----

// src (n0, n1, n2, L) with element strides (s0, s1, s2, 1) -> dst contiguous fp32
template <typename T>
__global__ void widen_kernel(const T *__restrict__ src, float *__restrict__ dst, int n1, int n2, int L, long long s0, long long s1,
                             long long s2, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int l = (int)(i % L);
    long long r = i / L;
    const int i2 = (int)(r % n2); r /= n2;
    const int i1 = (int)(r % n1); r /= n1;
    dst[i] = to_f32(src[r * s0 + i1 * s1 + i2 * s2 + l]);
  }
}
// src contiguous fp32 (n0, n1, L) -> dst with strides (s0, s1, 1)
template <typename T>
__global__ void narrow_kernel(const float *__restrict__ src, T *__restrict__ dst, int n1, int L, long long s0, long long s1, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int l = (int)(i % L);
    long long r = i / L;
    const int i1 = (int)(r % n1); r /= n1;
    dst[r * s0 + i1 * s1 + l] = from_f32<T>(src[i]);
  }
}
template <typename T>
static int widen(const void *src, float *dst, int n0, int n1, int n2, int L, long long s0, long long s1, long long s2, cudaStream_t st) {
  const long long total = (long long)n0 * n1 * n2 * L;
  widen_kernel<T><<<(unsigned)std::min<long long>((total + 255) / 256, kNumSMs * 16), 256, 0, st>>>((const T *)src, dst, n1, n2, L, s0, s1, s2, total);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}
template <typename T>
static int narrow_to(const float *src, void *dst, int n0, int n1, int L, long long s0, long long s1, cudaStream_t st) {
  const long long total = (long long)n0 * n1 * L;
  narrow_kernel<T><<<(unsigned)std::min<long long>((total + 255) / 256, kNumSMs * 16), 256, 0, st>>>(src, (T *)dst, n1, L, s0, s1, total);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

static bool widen_shape_ok(int dim, int L, int N, int G, int elem_bytes) {
  return elem_bytes == 2 && L % 8 != 0 && L % 4 == 0 && (N == 4 || N == 8 || N == 16) && (dim / G) % 32 == 0;
}
static size_t widen_fwd_bytes(int batch, int dim, int L, int N, int G) {
  return 3 * align256((size_t)batch * dim * L * 4) + 2 * align256((size_t)batch * G * N * L * 4);
}
static size_t widen_bwd_bytes(int batch, int dim, int L, int N, int G) {
  return 5 * align256((size_t)batch * dim * L * 4) + 2 * align256((size_t)batch * G * N * L * 4);
}
static sigma_scan_strides contiguous_strides(int dim, int L, int N, int G) {
  sigma_scan_strides st;
  st.u_batch = st.delta_batch = st.out_batch = (int64_t)dim * L;
  st.u_dim = st.delta_dim = st.out_dim = L;
  st.A_dim = N; st.A_dstate = 1;
  st.B_batch = st.C_batch = (int64_t)G * N * L;
  st.B_group = st.C_group = (int64_t)N * L;
  st.B_dstate = st.C_dstate = L;
  return st;
}

// which kernels a call runs: TMA-staged, TMA-staged on widened fp32 copies of 16-bit operands, or generic
enum { ROUTE_TMA = 0, ROUTE_WIDENED = 1, ROUTE_GENERIC = 2 };

template <typename T>
static int fwd_route(const void *u, const void *delta, const void *B, const void *C, const void *out, int batch, int dim, int L, int N,
                     int G, const sigma_scan_strides &s, const void *ws, size_t ws_bytes) {
  if (!force_generic() && scan_op_tma_eligible<T>(u, delta, B, C, out, dim, L, N, G, s)) return ROUTE_TMA;
  if (sizeof(T) == 2 && !force_generic() && widen_shape_ok(dim, L, N, G, 2) && ws != nullptr &&
      ws_bytes >= align256(scan_op_tma_workspace_bytes(batch, dim, N)) + widen_fwd_bytes(batch, dim, L, N, G) && s.A_dstate >= 0)
    return ROUTE_WIDENED;
  return ROUTE_GENERIC;
}

// `aligned`: dout / du / ddelta / dB / dC are 16-byte aligned (the other operands are checked by the eligibility test)
template <typename T>
static int bwd_route(bool aligned, const void *u, const void *delta, const void *B, const void *C, const void *du, int batch, int dim,
                     int L, int N, int G, size_t ws_bytes) {
  if (!force_generic() && aligned && scan_op_tma_eligible<T>(u, delta, B, C, du, dim, L, N, G, contiguous_strides(dim, L, N, G)))
    return ROUTE_TMA;
  if (sizeof(T) == 2 && !force_generic() && widen_shape_ok(dim, L, N, G, 2) &&
      ws_bytes >= align256(scan_op_bwd_tma_workspace_bytes(batch, dim, L, N, 4)) + widen_bwd_bytes(batch, dim, L, N, G))
    return ROUTE_WIDENED;
  return ROUTE_GENERIC;
}

template <typename T>
static int scan_fwd_dispatch(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                             const float *bias, void *out, float *x, int batch, int dim, int L, int N, int G, int softplus,
                             const sigma_scan_strides &s, void *ws, size_t ws_bytes, int force_split, cudaStream_t stream) {
  const int route = fwd_route<T>(u, delta, B, C, out, batch, dim, L, N, G, s, ws, ws_bytes);
  if (route == ROUTE_TMA)
    return scan_op_fwd_tma<T>(u, delta, A, B, C, D, bias, out, x, nullptr, batch, dim, L, N, G, softplus, s, ws, ws_bytes,
                              force_split, stream);
  if constexpr (sizeof(T) == 2) {
    const size_t core = align256(scan_op_tma_workspace_bytes(batch, dim, N));
    if (route == ROUTE_WIDENED) {
      char *w = (char *)ws + core;
      const size_t bdl = align256((size_t)batch * dim * L * 4), bgn = align256((size_t)batch * G * N * L * 4);
      float *u32 = (float *)w, *d32 = (float *)(w + bdl), *o32 = (float *)(w + 2 * bdl), *B32 = (float *)(w + 3 * bdl), *C32 = (float *)(w + 3 * bdl + bgn);
      int rc;
      if ((rc = widen<T>(u, u32, batch, dim, 1, L, s.u_batch, s.u_dim, 0, stream))) return rc;
      if ((rc = widen<T>(delta, d32, batch, dim, 1, L, s.delta_batch, s.delta_dim, 0, stream))) return rc;
      if ((rc = widen<T>(B, B32, batch, G, N, L, s.B_batch, s.B_group, s.B_dstate, stream))) return rc;
      if ((rc = widen<T>(C, C32, batch, G, N, L, s.C_batch, s.C_group, s.C_dstate, stream))) return rc;
      sigma_scan_strides cs = contiguous_strides(dim, L, N, G);
      cs.A_dim = s.A_dim; cs.A_dstate = s.A_dstate;
      if ((rc = scan_op_fwd_tma<float>(u32, d32, A, B32, C32, D, bias, o32, x, nullptr, batch, dim, L, N, G, softplus, cs, ws, core, force_split,
                                       stream))) return rc;
      return narrow_to<T>(o32, out, batch, dim, L, s.out_batch, s.out_dim, stream);
    }
  }
  return scan_op_fwd_generic<T>(u, delta, A, B, C, D, bias, out, x, nullptr, batch, dim, L, N, G, softplus, s, ws, ws_bytes,
                                force_split, stream);
}

template <typename T>
static int scan_bwd_dispatch(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                             const float *bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                             float *dD, float *dbias, int batch, int dim, int L, int N, int G, int softplus, void *ws,
                             size_t ws_bytes, int force_split, cudaStream_t stream, void *det_ws) {
  const sigma_scan_strides st = contiguous_strides(dim, L, N, G);
  const bool al = (((uintptr_t)dout | (uintptr_t)du | (uintptr_t)ddelta | (uintptr_t)dB | (uintptr_t)dC) & 15) == 0;
  const int route = bwd_route<T>(al, u, delta, B, C, du, batch, dim, L, N, G, ws_bytes);
  if (route == ROUTE_TMA)
    return scan_op_bwd_tma<T>(u, delta, A, B, C, D, bias, dout, du, ddelta, dA, dB, dC, dD, dbias, batch, dim, L, N, G, softplus,
                              ws, ws_bytes, force_split, stream, det_ws);
  if constexpr (sizeof(T) == 2) {
    const size_t core = align256(scan_op_bwd_tma_workspace_bytes(batch, dim, L, N, 4));
    if (route == ROUTE_WIDENED) {
      char *w = (char *)ws + core;
      const size_t bdl = align256((size_t)batch * dim * L * 4), bgn = align256((size_t)batch * G * N * L * 4);
      float *u32 = (float *)w, *d32 = (float *)(w + bdl), *g32 = (float *)(w + 2 * bdl), *du32 = (float *)(w + 3 * bdl), *dd32 = (float *)(w + 4 * bdl);
      float *B32 = (float *)(w + 5 * bdl), *C32 = (float *)(w + 5 * bdl + bgn);
      int rc;
      if ((rc = widen<T>(u, u32, batch, dim, 1, L, st.u_batch, st.u_dim, 0, stream))) return rc;
      if ((rc = widen<T>(delta, d32, batch, dim, 1, L, st.u_batch, st.u_dim, 0, stream))) return rc;
      if ((rc = widen<T>(dout, g32, batch, dim, 1, L, st.u_batch, st.u_dim, 0, stream))) return rc;
      if ((rc = widen<T>(B, B32, batch, G, N, L, st.B_batch, st.B_group, st.B_dstate, stream))) return rc;
      if ((rc = widen<T>(C, C32, batch, G, N, L, st.C_batch, st.C_group, st.C_dstate, stream))) return rc;
      if ((rc = scan_op_bwd_tma<float>(u32, d32, A, B32, C32, D, bias, g32, du32, dd32, dA, dB, dC, dD, dbias, batch, dim, L, N, G, softplus, ws,
                                       core, force_split, stream, det_ws))) return rc;
      if ((rc = narrow_to<T>(du32, du, batch, dim, L, st.u_batch, st.u_dim, stream))) return rc;
      return narrow_to<T>(dd32, ddelta, batch, dim, L, st.u_batch, st.u_dim, stream);
    }
  }
  return scan_op_bwd_generic<T>(u, delta, A, B, C, D, bias, dout, du, ddelta, dA, dB, dC, dD, dbias, batch, dim, L, N, G,
                                softplus, ws, ws_bytes, stream, det_ws);
}

// sigma_test_scan_plan for element type T: the route and plans the dispatchers above would pick for contiguous, 16-byte aligned
// operands and a workspace of ws_bytes.  sweep 0 = forward; 1 / 2 = backward / its deterministic build, whose kernels see
// ws_bytes (the partials of the deterministic build follow it).  out = {route, segments, tiles per segment, tiles, channels per
// CTA, ring stages, state-sweep segments, state-sweep tiles per segment}.
template <typename T>
static void scan_plan(int sweep, int batch, int dim, int L, int N, int G, int force_split, size_t ws_bytes, long long *out) {
  const void *al = (const void *)(uintptr_t)256;   // stands for any 16-byte aligned pointer
  const sigma_scan_strides st = contiguous_strides(dim, L, N, G);
  const int eb = (int)sizeof(T);
  ScanOpPlan main, state;
  int route;
  if (sweep == 0) {
    route = fwd_route<T>(al, al, al, al, al, batch, dim, L, N, G, st, ws_bytes ? al : nullptr, ws_bytes);
    if (route == ROUTE_GENERIC) main = scan_op_fwd_generic_plan(batch, dim, L, N, G, ws_bytes >= scan_op_workspace_bytes(batch, dim, N), force_split);
    else main = scan_op_fwd_tma_plan(route == ROUTE_TMA ? eb : 4, batch, dim, L, N, G, ws_bytes >= scan_op_tma_workspace_bytes(batch, dim, N), force_split);
    state.nsplit = state.tiles_per_split = 0;
  } else {
    route = bwd_route<T>(true, al, al, al, al, al, batch, dim, L, N, G, ws_bytes);
    if (route == ROUTE_GENERIC) {
      // one reverse walk per CTA after a serial state sweep (scan_op_bwd.cu): 32-position tiles, plain loads
      main.ntiles = (L + 31) / 32; main.nsplit = 1; main.tiles_per_split = main.ntiles; main.DT = 32; main.nst = 1;
      state = scan_op_fwd_generic_plan(batch, dim, L, N, G, false, 1);
    } else {
      const int e = route == ROUTE_TMA ? eb : 4;
      main = scan_op_bwd_tma_plan(e, batch, dim, L, N, G, force_split);
      state = scan_op_fwd_tma_plan(e, batch, dim, L, N, G, true, force_split);   // the workspace always holds its carries
    }
  }
  const long long v[8] = {route, main.nsplit, main.tiles_per_split, main.ntiles, main.DT, main.nst, state.nsplit, state.tiles_per_split};
  for (int i = 0; i < 8; ++i) out[i] = v[i];
}

}  // namespace sigma

using namespace sigma;

extern "C" {
#pragma GCC visibility push(default)

int sigma_abi_version(void) { return 2; }   // 2 removed sigma_ss2d_scan_bwd{,_split,_det}; additions only since 2
const char *sigma_last_error(void) { return g_err; }
uint64_t sigma_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

size_t sigma_scan_fwd_workspace_bytes(int batch, int dim, int seqlen, int dstate, int ngroups, int dtype) {
  // every element type is read natively: only the L-segment carries need scratch — plus, for 16-bit calls whose rows are not
  // 16-byte aligned but whose fp32 image is TMA-eligible, the widened operands
  size_t w = align256(std::max(scan_op_workspace_bytes(batch, dim, dstate), scan_op_tma_workspace_bytes(batch, dim, dstate)));
  if (dtype != SIGMA_F32 && widen_shape_ok(dim, seqlen, dstate, ngroups, 2)) w += widen_fwd_bytes(batch, dim, seqlen, dstate, ngroups);
  return w;
}

static int scan_fwd_entry(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                          const float *delta_bias, void *out, float *x, int batch, int dim, int seqlen, int dstate, int ngroups,
                          int dtype, int delta_softplus, const sigma_scan_strides *st, void *workspace, size_t workspace_bytes,
                          int force_split, cudaStream_t stream) {
  SIGMA_CHECK_ARG(u && delta && A && B && C && out && st, "sigma_scan_fwd: null pointer argument");
  SIGMA_CHECK_ARG(batch > 0 && dim > 0 && seqlen > 0 && dstate > 0 && ngroups > 0,
                  "sigma_scan_fwd: non-positive size (batch=%d dim=%d seqlen=%d dstate=%d ngroups=%d)",
                  batch, dim, seqlen, dstate, ngroups);
  SIGMA_CHECK_ARG(dstate <= 256, "sigma_scan_fwd: dstate=%d > 256 (selective_scan.cpp:198)", dstate);
  SIGMA_CHECK_ARG(dim % ngroups == 0, "sigma_scan_fwd: dim=%d not divisible by ngroups=%d", dim, ngroups);
  SIGMA_CHECK_ARG(dtype == SIGMA_F32 || dtype == SIGMA_F16 || dtype == SIGMA_BF16,
                  "sigma_scan_fwd: unknown dtype %d", dtype);
  SIGMA_CHECK_ARG(force_split >= 0, "sigma_scan_fwd_split: nsplit=%d < 0", force_split);
  if (dtype == SIGMA_F32)
    return scan_fwd_dispatch<float>(u, delta, A, B, C, D, delta_bias, out, x, batch, dim, seqlen, dstate, ngroups, delta_softplus,
                                    *st, workspace, workspace_bytes, force_split, stream);
  if (dtype == SIGMA_F16)
    return scan_fwd_dispatch<__half>(u, delta, A, B, C, D, delta_bias, out, x, batch, dim, seqlen, dstate, ngroups, delta_softplus,
                                     *st, workspace, workspace_bytes, force_split, stream);
  return scan_fwd_dispatch<__nv_bfloat16>(u, delta, A, B, C, D, delta_bias, out, x, batch, dim, seqlen, dstate, ngroups,
                                          delta_softplus, *st, workspace, workspace_bytes, force_split, stream);
}

int sigma_scan_fwd(const void *u, const void *delta, const float *A, const void *B, const void *C,
                   const float *D, const float *delta_bias, void *out, float *x, int batch, int dim,
                   int seqlen, int dstate, int ngroups, int dtype, int delta_softplus,
                   const sigma_scan_strides *st, void *workspace, size_t workspace_bytes, void *stream_) {
  return scan_fwd_entry(u, delta, A, B, C, D, delta_bias, out, x, batch, dim, seqlen, dstate, ngroups, dtype, delta_softplus, st,
                        workspace, workspace_bytes, 0, (cudaStream_t)stream_);
}

// test hook: force the number of L-segments of the forward, any dtype and route (nsplit = 0: the library's choice)
int sigma_scan_fwd_split(const void *u, const void *delta, const float *A, const void *B, const void *C,
                         const float *D, const float *delta_bias, void *out, float *x, int batch, int dim,
                         int seqlen, int dstate, int ngroups, int dtype, int delta_softplus,
                         const sigma_scan_strides *st, void *workspace, size_t workspace_bytes, int nsplit, void *stream_) {
  return scan_fwd_entry(u, delta, A, B, C, D, delta_bias, out, x, batch, dim, seqlen, dstate, ngroups, dtype, delta_softplus, st,
                        workspace, workspace_bytes, nsplit, (cudaStream_t)stream_);
}

// the launch plan of the op-level scan, host only (see include/sigma_b200.h)
int sigma_test_scan_plan(int sweep, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype, int nsplit,
                         size_t workspace_bytes, int64_t *out8_host) {
  SIGMA_CHECK_ARG(out8_host && sweep >= 0 && sweep <= 2 && batch > 0 && dim > 0 && seqlen > 0 && dstate > 0 && dstate <= 256 &&
                      ngroups > 0 && dim % ngroups == 0 && nsplit >= 0 &&
                      (dtype == SIGMA_F32 || dtype == SIGMA_F16 || dtype == SIGMA_BF16),
                  "sigma_test_scan_plan: bad arguments");
  if (sweep > 0 && dstate > 16) {   // the wide-state kernel: one walk per CTA after a serial state sweep, both sweeps alike
    const size_t need = sigma_scan_bwd_workspace_bytes(batch, dim, seqlen, dstate, ngroups, dtype);
    if (workspace_bytes < need) {
      set_error("sigma_scan_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
      return SIGMA_EWORKSPACE;
    }
    const ScanOpPlan main = scan_op_bwd_wide_plan(seqlen), state = scan_op_fwd_generic_plan(batch, dim, seqlen, dstate, ngroups, false, 1);
    const long long v[8] = {ROUTE_GENERIC, main.nsplit, main.tiles_per_split, main.ntiles, main.DT, main.nst, state.nsplit, state.tiles_per_split};
    for (int i = 0; i < 8; ++i) out8_host[i] = v[i];
    return SIGMA_OK;
  }
  if (sweep > 0) {   // what scan_bwd_entry checks before it dispatches
    const size_t base = sigma_scan_bwd_workspace_bytes(batch, dim, seqlen, dstate, ngroups, dtype);
    const size_t need = sweep == 2 ? sigma_scan_bwd_det_workspace_bytes(batch, dim, seqlen, dstate, ngroups, dtype) : base;
    if (workspace_bytes < need) {
      set_error("sigma_scan_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
      return SIGMA_EWORKSPACE;
    }
    if (sweep == 2) workspace_bytes = align256(base);
  }
  long long out[8];
  if (dtype == SIGMA_F32) scan_plan<float>(sweep, batch, dim, seqlen, dstate, ngroups, nsplit, workspace_bytes, out);
  else if (dtype == SIGMA_F16) scan_plan<__half>(sweep, batch, dim, seqlen, dstate, ngroups, nsplit, workspace_bytes, out);
  else scan_plan<__nv_bfloat16>(sweep, batch, dim, seqlen, dstate, ngroups, nsplit, workspace_bytes, out);
  for (int i = 0; i < 8; ++i) out8_host[i] = out[i];
  return SIGMA_OK;
}

#pragma GCC visibility pop
}  // extern "C"

// ---------------------------------------------------------------------------------------------
// fused channels-last pipeline
// ---------------------------------------------------------------------------------------------
namespace sigma {
static bool al16(const void *p) { return ((uintptr_t)p & 15) == 0; }
static bool al8(const void *p) { return ((uintptr_t)p & 7) == 0; }
// The row norms and the depthwise conv's output move 4 elements at a time: a pointer to elements of type t (SIGMA_F32,
// SIGMA_BF16, SIGMA_F16 or SIGMA_E4M3_ROWS) is aligned to 4 of them, 16 bytes for fp32, 8 for 16-bit and 4 for e4m3.  NULL passes.
static bool al4(const void *p, int t) {
  const uintptr_t bytes = t == SIGMA_F32 ? 16 : t == SIGMA_E4M3_ROWS ? 4 : 8;
  return ((uintptr_t)p & (bytes - 1)) == 0;
}

// The row-norm entry points share one checked body per operation shape.  fn names the entry point in every message; ti / to are
// the element types of the input rows (and z) and of the output.  e4m3 output (to = SIGMA_E4M3_ROWS) also writes each row's fp32
// scale to `scale`.  gamma, beta and gate are fp32.  Every check runs before the first CUDA call.

// LayerNorm of (rows, C) rows
static int layernorm_rows(const char *fn, int ti, int to, const void *x, const float *w, const float *b, void *y, float *scale,
                          int64_t rows, int C, float eps, void *stream) {
  SIGMA_CHECK_ARG(x && w && b && y && (to != SIGMA_E4M3_ROWS || scale), "%s: null pointer", fn);
  SIGMA_CHECK_ARG(C > 0 && C % 4 == 0 && rows >= 0, "%s: C=%d must be a positive multiple of 4", fn, C);
  SIGMA_CHECK_ARG(al4(x, ti) && al16(w) && al16(b) && al4(y, to), "%s: x, y must be aligned to 4 elements and w, b to 16 bytes", fn);
  RowNormParams p{(const float *)x, 0, 1, w, b, nullptr, 0, nullptr, (float *)y, rows, rows > 0 ? rows : 1, 0, 0, C, C, eps};
  p.qscale = scale;
  return row_norm_launch(ti, to, p, (cudaStream_t)stream);
}

// LayerNorm of an fp32 (batch, H, W, C) image's rows gathered by mode: 1 = PatchMerging2D's 2x2 blocks, rows of 4C; 2 = PatchExpand's
// pixel shuffle, each pixel's 4C channels as 4 rows of C stored at (batch, 2H, 2W, C)
static int layernorm_image(const char *fn, int mode, int to, const float *x, const float *w, const float *b, void *y, float *scale,
                           int batch, int H, int W, int C, float eps, void *stream) {
  SIGMA_CHECK_ARG(x && w && b && y && (to != SIGMA_E4M3_ROWS || scale), "%s: null pointer", fn);
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "%s: bad sizes", fn);
  SIGMA_CHECK_ARG(al16(x) && al16(w) && al16(b) && al4(y, to), "%s: x, w, b must be 16-byte and y 4-element aligned", fn);
  const int64_t rows = mode == 1 ? (int64_t)batch * ((H + 1) / 2) * ((W + 1) / 2) : (int64_t)batch * H * W * 4;
  const int D = mode == 1 ? 4 * C : C;
  RowNormParams p{x, 0, 1, w, b, nullptr, 0, nullptr, (float *)y, rows, rows, 0, 0, D, D, eps};
  p.mode = mode; p.gH = H; p.gW = W; p.qscale = scale;
  return row_norm_launch(SIGMA_F32, to, p, (cudaStream_t)stream);
}

// sum of K direction slabs -> LayerNorm [· SiLU(z)] [· gate]; e4m3 output merges K = 1 or 4 slabs
static int merge_norm_gate(const char *fn, int ti, int to, const void *y, int K, int64_t k_stride, int64_t in_batch_stride,
                           const float *gamma, const float *beta, const void *z, int64_t z_row_stride, const float *gate, void *out,
                           float *scale, int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch, int D,
                           float eps, void *stream) {
  const bool e4m3 = to == SIGMA_E4M3_ROWS;
  SIGMA_CHECK_ARG(y && gamma && beta && out && (!e4m3 || scale), "%s: null pointer", fn);
  SIGMA_CHECK_ARG((e4m3 ? K == 1 || K == 4 : K >= 1 && K <= 8) && D > 0 && D % 4 == 0 && rows >= 0 && rows_per_batch > 0,
                  "%s: bad sizes K=%d (%s) D=%d rows=%lld rows_per_batch=%lld", fn, K, e4m3 ? "1 or 4" : "1 to 8", D, (long long)rows,
                  (long long)rows_per_batch);
  SIGMA_CHECK_ARG(al4(y, ti) && al4(z, ti) && al4(out, to) && al16(gamma) && al16(beta) && al16(gate) && k_stride % 4 == 0 &&
                      in_batch_stride % 4 == 0 && out_batch_stride % 4 == 0 && out_row_stride % 4 == 0 && z_row_stride % 4 == 0,
                  "%s: y / z / out must be 4-element and gamma / beta / gate 16-byte aligned, strides multiples of 4", fn);
  RowNormParams p{(const float *)y, k_stride, K, gamma, beta, (const float *)z, z_row_stride, gate, (float *)out, rows, rows_per_batch,
                  in_batch_stride, out_batch_stride, out_row_stride, D, eps};
  p.qscale = scale;
  return row_norm_launch(ti, to, p, (cudaStream_t)stream);
}

// LayerNorm backward, x / dy / dx of element type dtype; det: the deterministic build in `workspace`
static int layernorm_bwd_checked(const char *fn, int dtype, const void *x, const void *dy, const float *w, void *dx, float *dw, float *db,
                                 int64_t rows, int C, float eps, void *stream, bool det = false, void *workspace = nullptr,
                                 size_t workspace_bytes = 0) {
  SIGMA_CHECK_ARG(x && dy && w && dx && dw && db, "%s: null pointer", fn);
  SIGMA_CHECK_ARG(C > 0 && C % 4 == 0 && rows >= 0, "%s: C=%d must be a positive multiple of 4", fn, C);
  SIGMA_CHECK_ARG(al4(x, dtype) && al4(dy, dtype) && al4(dx, dtype) && al16(w), "%s: x, dy, dx must be 4-element and w 16-byte aligned",
                  fn);
  if (det) {
    const size_t need = layernorm_bwd_det_workspace_bytes(rows, C);
    SIGMA_CHECK_ARG(workspace != nullptr && al16(workspace) && workspace_bytes >= need,
                    "%s: needs %zu 16-byte aligned workspace bytes, got %zu", fn, need, workspace_bytes);
  }
  return layernorm_bwd_launch(dtype, x, dy, w, dx, dw, db, rows, C, eps, (cudaStream_t)stream, det ? (float *)workspace : nullptr);
}

static int dwconv3x3_silu_fwd_any(const char *fn, int dtype, const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w,
                                  const float *bias, void *y, int64_t y_batch_stride, int batch, int H, int W, int D, void *stream) {
  const int q = dtype == SIGMA_F32 ? 4 : 8;   // elements per 16 bytes
  SIGMA_CHECK_ARG(x && w && y, "%s: null pointer", fn);
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && D > 0 && D % 4 == 0, "%s: bad sizes", fn);
  SIGMA_CHECK_ARG(al16(x) && al4(y, dtype) && x_row_stride % q == 0 && x_batch_stride % q == 0 && y_batch_stride % 4 == 0,
                  "%s: x must be 16-byte aligned with strides multiples of %d elements (TMA), y 4-element aligned", fn, q);
  return dwconv3x3_silu_fwd_launch(dtype, x, x_row_stride, x_batch_stride, w, bias, y, y_batch_stride, batch, H, W, D,
                                   (cudaStream_t)stream);
}
}  // namespace sigma

extern "C" {
#pragma GCC visibility push(default)

static int linear_16bit(const char *fn, int dtype, const void *A, int64_t lda, const void *W, const float *bias, const float *residual,
                        int64_t ldr, const float *rscale, void *C, int64_t ldc, int c_dtype, int64_t M, int N, int K, void *stream) {
  const bool f16 = dtype == SIGMA_F16;
  SIGMA_CHECK_ARG(A && W && C, "%s: null pointer", fn);
  SIGMA_CHECK_ARG(c_dtype == SIGMA_F32 || c_dtype == dtype, "%s: c_dtype %d (SIGMA_F32 or %s)", fn, c_dtype, f16 ? "SIGMA_F16" : "SIGMA_BF16");
  SIGMA_CHECK_ARG(M >= 0 && M < (1LL << 31) && N > 0 && K > 0, "%s: bad sizes M=%lld N=%d K=%d", fn, (long long)M, N, K);
  SIGMA_CHECK_ARG(K % 8 == 0 && lda % 8 == 0 && N % 4 == 0 && ldc % 4 == 0 && (residual == nullptr || ldr % 4 == 0) && lda >= K && ldc >= N,
                  "%s: K and lda must be multiples of 8 (16-byte %s TMA rows); N, ldc, ldr multiples of 4", fn, f16 ? "fp16" : "bf16");
  SIGMA_CHECK_ARG(al16(A) && al16(W) && al16(C) && al16(bias) && al16(residual) && al16(rscale), "%s: pointers must be 16-byte aligned", fn);
  SIGMA_CHECK_ARG(rscale == nullptr || residual != nullptr, "%s: rscale without residual", fn);
  return gemm_launch(f16 ? GemmOp::F16 : GemmOp::BF16, A, lda, W, nullptr, nullptr, nullptr, bias, residual, ldr, rscale, C, ldc,
                     c_dtype == dtype, M, N, K, (cudaStream_t)stream);
}

int sigma_layernorm_fwd(const float *x, const float *w, const float *b, float *y, int64_t rows, int C, float eps,
                        void *stream) {
  return layernorm_rows("sigma_layernorm_fwd", SIGMA_F32, SIGMA_F32, x, w, b, y, nullptr, rows, C, eps, stream);
}

int sigma_layernorm_fwd_bf16(const float *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream) {
  return layernorm_rows("sigma_layernorm_fwd_bf16", SIGMA_F32, SIGMA_BF16, x, w, b, y, nullptr, rows, C, eps, stream);
}

int sigma_layernorm_fwd_fp16(const float *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream) {
  return layernorm_rows("sigma_layernorm_fwd_fp16", SIGMA_F32, SIGMA_F16, x, w, b, y, nullptr, rows, C, eps, stream);
}

int sigma_layernorm_fwd_fp8(const float *x, const float *w, const float *b, void *q, float *scale, int64_t rows, int C, float eps,
                            void *stream) {
  return layernorm_rows("sigma_layernorm_fwd_fp8", SIGMA_F32, SIGMA_E4M3_ROWS, x, w, b, q, scale, rows, C, eps, stream);
}

int sigma_layernorm_fwd_bf16io(const void *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream) {
  return layernorm_rows("sigma_layernorm_fwd_bf16io", SIGMA_BF16, SIGMA_BF16, x, w, b, y, nullptr, rows, C, eps, stream);
}

// the fp16 training mode: x and y fp16 (merge + norm + gate's fp16 in / out instance with one input and no gate)
int sigma_layernorm_fwd_fp16io(const void *x, const float *w, const float *b, void *y, int64_t rows, int C, float eps, void *stream) {
  return layernorm_rows("sigma_layernorm_fwd_fp16io", SIGMA_F16, SIGMA_F16, x, w, b, y, nullptr, rows, C, eps, stream);
}

int sigma_layernorm_bwd(const float *x, const float *dy, const float *w, float *dx, float *dw, float *db, int64_t rows, int C, float eps,
                        void *stream) {
  return layernorm_bwd_checked("sigma_layernorm_bwd", SIGMA_F32, x, dy, w, dx, dw, db, rows, C, eps, stream);
}

int sigma_layernorm_bwd_bf16(const void *x, const void *dy, const float *w, void *dx, float *dw, float *db, int64_t rows, int C, float eps,
                             void *stream) {
  return layernorm_bwd_checked("sigma_layernorm_bwd_bf16", SIGMA_BF16, x, dy, w, dx, dw, db, rows, C, eps, stream);
}

int sigma_layernorm_bwd_fp16(const void *x, const void *dy, const float *w, void *dx, float *dw, float *db, int64_t rows, int C, float eps,
                             void *stream) {
  return layernorm_bwd_checked("sigma_layernorm_bwd_fp16", SIGMA_F16, x, dy, w, dx, dw, db, rows, C, eps, stream);
}

size_t sigma_layernorm_bwd_det_workspace_bytes(int64_t rows, int C) {
  if (rows < 0 || C <= 0 || C % 4) return 0;
  return layernorm_bwd_det_workspace_bytes(rows, C);
}

int sigma_layernorm_bwd_det(const float *x, const float *dy, const float *w, float *dx, float *dw, float *db, int64_t rows, int C, float eps,
                            void *workspace, size_t workspace_bytes, void *stream) {
  return layernorm_bwd_checked("sigma_layernorm_bwd_det", SIGMA_F32, x, dy, w, dx, dw, db, rows, C, eps, stream, true, workspace,
                               workspace_bytes);
}

int sigma_upsample_bilinear_bwd(const float *dy, float *dx, int batch, int C, int Hin, int Win, int Hout, int Wout, float ratio_h,
                                float ratio_w, int channels_last, void *stream) {
  SIGMA_CHECK_ARG(dy && dx, "sigma_upsample_bilinear_bwd: null pointer");
  SIGMA_CHECK_ARG(batch > 0 && C > 0 && Hin > 0 && Win > 0 && Hout > 0 && Wout > 0, "sigma_upsample_bilinear_bwd: bad sizes");
  SIGMA_CHECK_ARG(ratio_h > 0.f && ratio_w > 0.f, "sigma_upsample_bilinear_bwd: ratios must be positive");
  return upsample_bilinear_bwd_launch(dy, dx, batch, C, Hin, Win, Hout, Wout, ratio_h, ratio_w, channels_last, (cudaStream_t)stream);
}

int sigma_patch_merge_norm_fwd(const float *x, const float *w, const float *b, float *y, int batch, int H, int W, int C,
                               float eps, void *stream) {
  return layernorm_image("sigma_patch_merge_norm_fwd", 1, SIGMA_F32, x, w, b, y, nullptr, batch, H, W, C, eps, stream);
}

int sigma_patch_merge_norm_fwd_bf16(const float *x, const float *w, const float *b, void *y, int batch, int H, int W, int C,
                                    float eps, void *stream) {
  return layernorm_image("sigma_patch_merge_norm_fwd_bf16", 1, SIGMA_BF16, x, w, b, y, nullptr, batch, H, W, C, eps, stream);
}

int sigma_patch_merge_norm_fwd_fp16(const float *x, const float *w, const float *b, void *y, int batch, int H, int W, int C,
                                    float eps, void *stream) {
  return layernorm_image("sigma_patch_merge_norm_fwd_fp16", 1, SIGMA_F16, x, w, b, y, nullptr, batch, H, W, C, eps, stream);
}

int sigma_patch_merge_norm_fwd_fp8(const float *x, const float *w, const float *b, void *q, float *scale, int batch, int H, int W, int C,
                                   float eps, void *stream) {
  return layernorm_image("sigma_patch_merge_norm_fwd_fp8", 1, SIGMA_E4M3_ROWS, x, w, b, q, scale, batch, H, W, C, eps, stream);
}

int sigma_pixel_shuffle_norm_fwd(const float *x, const float *w, const float *b, float *y, int batch, int H, int W, int C,
                                 float eps, void *stream) {
  return layernorm_image("sigma_pixel_shuffle_norm_fwd", 2, SIGMA_F32, x, w, b, y, nullptr, batch, H, W, C, eps, stream);
}

int sigma_merge_norm_gate_fwd(const float *y, int K, int64_t k_stride, int64_t in_batch_stride, const float *gamma,
                              const float *beta, const float *z, int64_t z_row_stride, const float *gate, float *out,
                              int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch,
                              int D, float eps, void *stream) {
  return merge_norm_gate("sigma_merge_norm_gate_fwd", SIGMA_F32, SIGMA_F32, y, K, k_stride, in_batch_stride, gamma, beta, z, z_row_stride,
                         gate, out, nullptr, out_batch_stride, out_row_stride, rows, rows_per_batch, D, eps, stream);
}

int sigma_merge_norm_gate_fwd_fp8(const void *y, int K, int64_t k_stride, int64_t in_batch_stride, const float *gamma,
                                  const float *beta, const void *z, int64_t z_row_stride, const float *gate, void *q, float *scale,
                                  int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch,
                                  int D, float eps, void *stream) {
  return merge_norm_gate("sigma_merge_norm_gate_fwd_fp8", SIGMA_BF16, SIGMA_E4M3_ROWS, y, K, k_stride, in_batch_stride, gamma, beta, z,
                         z_row_stride, gate, q, scale, out_batch_stride, out_row_stride, rows, rows_per_batch, D, eps, stream);
}

int sigma_merge_norm_gate_fwd_bf16(const void *y, int K, int64_t k_stride, int64_t in_batch_stride, const float *gamma,
                                   const float *beta, const void *z, int64_t z_row_stride, const float *gate, void *out,
                                   int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch,
                                   int D, float eps, void *stream) {
  return merge_norm_gate("sigma_merge_norm_gate_fwd_bf16", SIGMA_BF16, SIGMA_BF16, y, K, k_stride, in_batch_stride, gamma, beta, z,
                         z_row_stride, gate, out, nullptr, out_batch_stride, out_row_stride, rows, rows_per_batch, D, eps, stream);
}

int sigma_merge_norm_gate_fwd_fp16(const void *y, int K, int64_t k_stride, int64_t in_batch_stride, const float *gamma,
                                   const float *beta, const void *z, int64_t z_row_stride, const float *gate, void *out,
                                   int64_t out_batch_stride, int64_t out_row_stride, int64_t rows, int64_t rows_per_batch,
                                   int D, float eps, void *stream) {
  return merge_norm_gate("sigma_merge_norm_gate_fwd_fp16", SIGMA_F16, SIGMA_F16, y, K, k_stride, in_batch_stride, gamma, beta, z,
                         z_row_stride, gate, out, nullptr, out_batch_stride, out_row_stride, rows, rows_per_batch, D, eps, stream);
}

int sigma_dwconv3x3_silu_fwd(const float *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w,
                             const float *bias, float *y, int64_t y_batch_stride, int batch, int H, int W, int D,
                             void *stream) {
  return dwconv3x3_silu_fwd_any("sigma_dwconv3x3_silu_fwd", SIGMA_F32, x, x_row_stride, x_batch_stride, w, bias, y, y_batch_stride, batch,
                                H, W, D, stream);
}

int sigma_dwconv3x3_silu_fwd_bf16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  void *y, int64_t y_batch_stride, int batch, int H, int W, int D, void *stream) {
  return dwconv3x3_silu_fwd_any("sigma_dwconv3x3_silu_fwd_bf16", SIGMA_BF16, x, x_row_stride, x_batch_stride, w, bias, y,
                                y_batch_stride, batch, H, W, D, stream);
}

int sigma_dwconv3x3_silu_fwd_fp16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  void *y, int64_t y_batch_stride, int batch, int H, int W, int D, void *stream) {
  return dwconv3x3_silu_fwd_any("sigma_dwconv3x3_silu_fwd_fp16", SIGMA_F16, x, x_row_stride, x_batch_stride, w, bias, y,
                                y_batch_stride, batch, H, W, D, stream);
}

size_t sigma_dwconv3x3_silu_bwd_workspace_bytes(int batch, int H, int W, int D) {
  if (batch <= 0 || H <= 0 || W <= 0 || D <= 0) return 0;
  return dwconv3x3_silu_bwd_workspace_bytes(batch, H, W, D);
}

static int dwconv3x3_silu_bwd_any(const char *fn, int dtype, const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w,
                                  const float *bias, const void *dy, int64_t dy_batch_stride, void *dx, int64_t dx_batch_stride, float *dw,
                                  float *dbias, int batch, int H, int W, int D, void *workspace, size_t workspace_bytes, void *stream) {
  const int q = dtype == SIGMA_F32 ? 4 : 8;   // elements per 16 bytes
  SIGMA_CHECK_ARG(x && w && dy && dx && dw, "%s: null pointer", fn);
  SIGMA_CHECK_ARG((bias == nullptr) == (dbias == nullptr), "%s: bias and dbias must be given together (or both NULL)", fn);
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && D > 0 && D % q == 0, "%s: bad sizes batch=%d H=%d W=%d D=%d (D %% %d == 0)", fn, batch,
                  H, W, D, q);
  SIGMA_CHECK_ARG(al16(x) && al16(dy) && al16(dx) && x_row_stride % q == 0 && x_batch_stride % q == 0 && dy_batch_stride % q == 0 &&
                      dx_batch_stride % q == 0,
                  "%s: x, dy, dx must be 16-byte aligned with strides multiples of %d elements (TMA)", fn, q);
  const size_t need = dwconv3x3_silu_bwd_workspace_bytes(batch, H, W, D);
  SIGMA_CHECK_ARG(workspace != nullptr && al16(workspace) && workspace_bytes >= need,
                  "%s: needs %zu 16-byte aligned workspace bytes, got %zu", fn, need, workspace_bytes);
  return dwconv3x3_silu_bwd_launch(dtype, x, x_row_stride, x_batch_stride, w, bias, dy, dy_batch_stride, dx, dx_batch_stride, dw, dbias,
                                   batch, H, W, D, workspace, (cudaStream_t)stream);
}

int sigma_dwconv3x3_silu_bwd(const float *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                             const float *dy, int64_t dy_batch_stride, float *dx, int64_t dx_batch_stride, float *dw, float *dbias,
                             int batch, int H, int W, int D, void *workspace, size_t workspace_bytes, void *stream) {
  return dwconv3x3_silu_bwd_any("sigma_dwconv3x3_silu_bwd", SIGMA_F32, x, x_row_stride, x_batch_stride, w, bias, dy, dy_batch_stride, dx,
                                dx_batch_stride, dw, dbias, batch, H, W, D, workspace, workspace_bytes, stream);
}

int sigma_dwconv3x3_silu_bwd_bf16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  const void *dy, int64_t dy_batch_stride, void *dx, int64_t dx_batch_stride, float *dw, float *dbias,
                                  int batch, int H, int W, int D, void *workspace, size_t workspace_bytes, void *stream) {
  return dwconv3x3_silu_bwd_any("sigma_dwconv3x3_silu_bwd_bf16", SIGMA_BF16, x, x_row_stride, x_batch_stride, w, bias, dy, dy_batch_stride,
                                dx, dx_batch_stride, dw, dbias, batch, H, W, D, workspace, workspace_bytes, stream);
}

int sigma_dwconv3x3_silu_bwd_fp16(const void *x, int64_t x_row_stride, int64_t x_batch_stride, const float *w, const float *bias,
                                  const void *dy, int64_t dy_batch_stride, void *dx, int64_t dx_batch_stride, float *dw, float *dbias,
                                  int batch, int H, int W, int D, void *workspace, size_t workspace_bytes, void *stream) {
  return dwconv3x3_silu_bwd_any("sigma_dwconv3x3_silu_bwd_fp16", SIGMA_F16, x, x_row_stride, x_batch_stride, w, bias, dy, dy_batch_stride,
                                dx, dx_batch_stride, dw, dbias, batch, H, W, D, workspace, workspace_bytes, stream);
}

int sigma_ss2d_padded_cp(int N, int R) {
  const int rp = pad_rp(R);
  return rp < 0 ? -1 : 2 * N + rp;
}

size_t sigma_ss2d_scan_workspace_bytes(int kind, int batch, int H, int W, int D, int N) {
  (void)H; (void)W;
  return ss2d_scan_workspace_bytes(kind, batch, D, N);
}

static int ss2d_check(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                      const float *Ds, float *y, int batch, int H, int W, int D, int N, int R, int Cp) {
  SIGMA_CHECK_ARG(xc && xdbl && dtw && dtb && A && Ds && y, "sigma_ss2d_scan_fwd: null pointer");
  SIGMA_CHECK_ARG(kind == SIGMA_DIRS_CROSS4 || kind == SIGMA_DIRS_SEQ2 || kind == SIGMA_DIRS_CROSS,
                  "sigma_ss2d_scan_fwd: unknown kind %d", kind);
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && D > 0 && D % 4 == 0 && R > 0, "sigma_ss2d_scan_fwd: bad sizes");
  SIGMA_CHECK_ARG(kind != SIGMA_DIRS_CROSS || batch % 2 == 0, "sigma_ss2d_scan_fwd: CROSS needs batch = 2·images");
  SIGMA_CHECK_ARG(N == 4 || N == 8 || N == 16, "sigma_ss2d_scan_fwd: d_state=%d unsupported (4, 8, 16)", N);
  SIGMA_CHECK_ARG(Cp == sigma_ss2d_padded_cp(N, R), "sigma_ss2d_scan_fwd: Cp=%d must equal sigma_ss2d_padded_cp(N=%d, R=%d)=%d",
                  Cp, N, R, sigma_ss2d_padded_cp(N, R));
  SIGMA_CHECK_ARG(al16(xc) && al16(xdbl) && al16(y), "sigma_ss2d_scan_fwd: xc / xdbl / y must be 16-byte aligned");
  return SIGMA_OK;
}

static int ss2d_scan_fwd_16bit(const char *fn, int dtype, int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb,
                               const float *A, const float *Ds, void *y, int batch, int H, int W, int D, int N, int R, int Cp,
                               void *workspace, size_t workspace_bytes, void *stream) {
  int rc = ss2d_check(kind, (const float *)xc, xdbl, dtw, dtb, A, Ds, (float *)y, batch, H, W, D, N, R, Cp);
  if (rc) return rc;
  SIGMA_CHECK_ARG(D % 8 == 0, "%s: D=%d must be a multiple of 8 (16-byte TMA rows)", fn, D);
  return ss2d_scan_fwd(kind, (const float *)xc, xdbl, dtw, dtb, A, Ds, (float *)y, batch, H, W, D, N, R, Cp, workspace, workspace_bytes,
                       0, (cudaStream_t)stream, nullptr, nullptr, dtype);
}

int sigma_ss2d_scan_fwd(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb,
                        const float *A, const float *Ds, float *y, int batch, int H, int W, int D, int N, int R, int Cp,
                        void *workspace, size_t workspace_bytes, void *stream) {
  int rc = ss2d_check(kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp);
  if (rc) return rc;
  return ss2d_scan_fwd(kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp, workspace, workspace_bytes, 0,
                       (cudaStream_t)stream);
}

int sigma_ss2d_scan_fwd_bf16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                             const float *Ds, void *y, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                             size_t workspace_bytes, void *stream) {
  return ss2d_scan_fwd_16bit("sigma_ss2d_scan_fwd_bf16", SIGMA_BF16, kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp,
                             workspace, workspace_bytes, stream);
}

int sigma_ss2d_scan_fwd_fp16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                             const float *Ds, void *y, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                             size_t workspace_bytes, void *stream) {
  return ss2d_scan_fwd_16bit("sigma_ss2d_scan_fwd_fp16", SIGMA_F16, kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp,
                             workspace, workspace_bytes, stream);
}

// test hook: force the number of L-segments
int sigma_ss2d_scan_fwd_split(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb,
                              const float *A, const float *Ds, float *y, int batch, int H, int W, int D, int N, int R,
                              int Cp, void *workspace, size_t workspace_bytes, int nsplit, void *stream) {
  int rc = ss2d_check(kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp);
  if (rc) return rc;
  return ss2d_scan_fwd(kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp, workspace, workspace_bytes, nsplit,
                       (cudaStream_t)stream);
}

// test hooks (host logic only, no CUDA call): the launch heuristics, so that CPU tests can hold them to the recorded sweeps
int sigma_test_pick_segments(int64_t ctas, int warps_per_cta, int ntiles, int N) { return ss2d_pick_segments_hook(ctas, warps_per_cta, ntiles, N); }
int sigma_test_pick_bn(int N, int64_t m_tiles) { return gemm_pick_bn_hook(N, m_tiles); }
// the launch plan of sigma_linear_tf32{,x3} (conv_B = 0) or of sigma_conv3x3_tf32 (conv_B > 0: input (conv_B, conv_H, conv_W, K),
// N output channels), SIGMA_GEMM_BN included: out6_host = {tile width, ring stages, grid, tiles, shared-memory bytes, CTAs per SM}
int sigma_test_gemm_plan(int64_t M, int N, int K, int x3, int conv_B, int conv_H, int conv_W, int64_t *out6_host) {
  SIGMA_CHECK_ARG(out6_host && N > 0 && K > 0 && (conv_B > 0 ? conv_H > 0 && conv_W > 0 : M > 0), "sigma_test_gemm_plan: bad arguments");
  long long out[6];
  const int rc = gemm_plan_hook(M, N, K, x3, conv_B, conv_H, conv_W, out);
  if (rc) return rc;
  for (int i = 0; i < 6; ++i) out6_host[i] = out[i];
  return SIGMA_OK;
}

// the L-segment plan of sigma_ss2d_scan_bwd_saved{,_bf16,_det} (nsplit = 0: the library's choice):
// out4_host = {segments, tiles per segment, tiles of the longest walk, tiles of the shortest walk}
int sigma_test_ss2d_bwd_plan(int kind, int batch, int H, int W, int D, int N, int nsplit, int64_t *out4_host) {
  SIGMA_CHECK_ARG(out4_host && (kind == SIGMA_DIRS_CROSS4 || kind == SIGMA_DIRS_SEQ2 || kind == SIGMA_DIRS_CROSS) && batch > 0 && H > 0 &&
                      W > 0 && D > 0 && D % 64 == 0 && (N == 4 || N == 16) && nsplit >= 0 && (kind != SIGMA_DIRS_CROSS || batch % 2 == 0),
                  "sigma_test_ss2d_bwd_plan: bad arguments");
  long long out[4];
  const int rc = ss2d_bwd_plan_hook(kind, batch, H, W, D, N, nsplit, out);
  if (rc) return rc;
  for (int i = 0; i < 4; ++i) out4_host[i] = out[i];
  return SIGMA_OK;
}

// the launch plan of sigma_ss2d_scan_fwd{,_split,_bf16}, with bf16 = 2 of sigma_ss2d_scan_fwd_save_bf16, with bf16 = 3 of
// sigma_ss2d_scan_fwd_fp16 and with bf16 = 4 of sigma_ss2d_scan_fwd_save_fp16 (force_split = 0: the library's choice), environment
// overrides included:
// out8_host = {segments, tiles per segment, tiles of the longest walk, of the shortest, warps per CTA, ring depth, register
// budget (CTAs per SM the kernel build assumes), dynamic shared-memory bytes}
int sigma_test_ss2d_fwd_plan(int kind, int batch, int H, int W, int D, int N, int R, int bf16, int force_split, size_t workspace_bytes,
                             int64_t *out8_host) {
  SIGMA_CHECK_ARG(out8_host && (kind == SIGMA_DIRS_CROSS4 || kind == SIGMA_DIRS_SEQ2 || kind == SIGMA_DIRS_CROSS) && batch > 0 &&
                      H > 0 && W > 0 && D > 0 && D % (bf16 ? 8 : 4) == 0 && R > 0 && force_split >= 0 &&
                      (kind != SIGMA_DIRS_CROSS || batch % 2 == 0),
                  "sigma_test_ss2d_fwd_plan: bad arguments");
  if ((bf16 == 2 || bf16 == 4) && N != 4 && N != 16) {
    set_error("sigma_test_ss2d_fwd_plan: d_state=%d unsupported by the %s training forward (4, 16)", N, bf16 == 4 ? "fp16" : "bf16");
    return SIGMA_EUNSUPPORTED;
  }
  long long out[8];
  const int rc = ss2d_fwd_plan_hook(kind, batch, H, W, D, N, R, bf16 == 3 || bf16 == 4 ? SIGMA_F16 : bf16 ? SIGMA_BF16 : SIGMA_F32,
                                    force_split, workspace_bytes, out);
  if (rc) return rc;
  for (int i = 0; i < 8; ++i) out8_host[i] = out[i];
  return SIGMA_OK;
}

// training forward: the forward plus what the fused backward needs (delta' slabs, block-start states)
size_t sigma_ss2d_scan_hs_bytes(int kind, int batch, int H, int W, int D, int N) {
  if (kind != SIGMA_DIRS_CROSS4 && kind != SIGMA_DIRS_SEQ2 && (kind != SIGMA_DIRS_CROSS || batch % 2)) return 0;
  return ss2d_scan_hs_bytes(kind, batch, H, W, D, N);
}

int sigma_ss2d_scan_fwd_save(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                             const float *Ds, float *y, float *delta, float *hs, int batch, int H, int W, int D, int N, int R, int Cp,
                             void *workspace, size_t workspace_bytes, int nsplit, void *stream) {
  int rc = ss2d_check(kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp);
  if (rc) return rc;
  SIGMA_CHECK_ARG(delta && hs && al16(delta) && al16(hs), "sigma_ss2d_scan_fwd_save: delta / hs must be non-null and 16-byte aligned");
  SIGMA_CHECK_ARG(kind == SIGMA_DIRS_CROSS4 || kind == SIGMA_DIRS_SEQ2 || kind == SIGMA_DIRS_CROSS,
                  "sigma_ss2d_scan_fwd_save: kind %d unsupported (CROSS4, SEQ2, CROSS)", kind);
  SIGMA_CHECK_ARG(N == 4 || N == 16, "sigma_ss2d_scan_fwd_save: d_state=%d unsupported (4, 16)", N);
  return ss2d_scan_fwd(kind, xc, xdbl, dtw, dtb, A, Ds, y, batch, H, W, D, N, R, Cp, workspace, workspace_bytes, nsplit,
                       (cudaStream_t)stream, delta, hs);
}

// The bf16 and fp16 training modes share a body: `fn` names the entry point in its error strings, dtype is SIGMA_BF16 or SIGMA_F16.
// xc, y and delta are 16-bit, and delta is rounded before the recurrence uses it.
static int ss2d_scan_fwd_save_16bit(const char *fn, int dtype, int kind, const void *xc, const float *xdbl, const float *dtw,
                                    const float *dtb, const float *A, const float *Ds, void *y, void *delta, float *hs, int batch, int H,
                                    int W, int D, int N, int R, int Cp, void *workspace, size_t workspace_bytes, int nsplit, void *stream) {
  if (N == 8) {
    set_error("%s: d_state=8 unsupported (4, 16)", fn);
    return SIGMA_EUNSUPPORTED;
  }
  int rc = ss2d_check(kind, (const float *)xc, xdbl, dtw, dtb, A, Ds, (float *)y, batch, H, W, D, N, R, Cp);
  if (rc) return rc;
  SIGMA_CHECK_ARG(D % 8 == 0, "%s: D=%d must be a multiple of 8 (16-byte TMA rows)", fn, D);
  SIGMA_CHECK_ARG(delta && hs && al16(delta) && al16(hs), "%s: delta / hs must be non-null and 16-byte aligned", fn);
  SIGMA_CHECK_ARG(nsplit >= 0, "%s: nsplit=%d < 0", fn, nsplit);
  return ss2d_scan_fwd(kind, (const float *)xc, xdbl, dtw, dtb, A, Ds, (float *)y, batch, H, W, D, N, R, Cp, workspace, workspace_bytes,
                       nsplit, (cudaStream_t)stream, (float *)delta, hs, dtype);
}

int sigma_ss2d_scan_fwd_save_bf16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                  const float *Ds, void *y, void *delta, float *hs, int batch, int H, int W, int D, int N, int R, int Cp,
                                  void *workspace, size_t workspace_bytes, int nsplit, void *stream) {
  return ss2d_scan_fwd_save_16bit("sigma_ss2d_scan_fwd_save_bf16", SIGMA_BF16, kind, xc, xdbl, dtw, dtb, A, Ds, y, delta, hs, batch, H, W,
                                  D, N, R, Cp, workspace, workspace_bytes, nsplit, stream);
}

int sigma_ss2d_scan_fwd_save_fp16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                  const float *Ds, void *y, void *delta, float *hs, int batch, int H, int W, int D, int N, int R, int Cp,
                                  void *workspace, size_t workspace_bytes, int nsplit, void *stream) {
  return ss2d_scan_fwd_save_16bit("sigma_ss2d_scan_fwd_save_fp16", SIGMA_F16, kind, xc, xdbl, dtw, dtb, A, Ds, y, delta, hs, batch, H, W,
                                  D, N, R, Cp, workspace, workspace_bytes, nsplit, stream);
}

size_t sigma_ss2d_scan_bwd_workspace_bytes(int kind, int batch, int H, int W, int D, int N) {
  if (kind != SIGMA_DIRS_CROSS4 && kind != SIGMA_DIRS_SEQ2 && (kind != SIGMA_DIRS_CROSS || batch % 2)) return 0;
  return ss2d_scan_bwd_workspace_bytes(kind, batch, H, W, D, N);
}

// no deterministic build of kind CROSS: under torch.use_deterministic_algorithms(True) CroMB trains through the op-level _det kernels
size_t sigma_ss2d_scan_bwd_det_workspace_bytes(int kind, int batch, int H, int W, int D, int N) {
  if ((kind != SIGMA_DIRS_CROSS4 && kind != SIGMA_DIRS_SEQ2) || (N != 4 && N != 16) || D % 64) return 0;
  return ss2d_scan_bwd_det_workspace_bytes(kind, batch, H, W, D, N);
}

static int ss2d_bwd_entry(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A, const float *Ds,
                          const float *dy, const float *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl, float *dA,
                          float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *ws, size_t wsb, int nsplit,
                          void *stream, int det = 0, int xdtype = SIGMA_F32) {
  SIGMA_CHECK_ARG(xc && xdbl && dtw && dtb && A && Ds && dy && delta && dxc && ddelta && dxdbl && dA && dDs && ddtb,
                  "sigma_ss2d_scan_bwd_saved: null pointer");
  SIGMA_CHECK_ARG(kind == SIGMA_DIRS_CROSS4 || kind == SIGMA_DIRS_SEQ2 || kind == SIGMA_DIRS_CROSS,
                  "sigma_ss2d_scan_bwd_saved: kind %d unsupported (CROSS4, SEQ2, CROSS)", kind);
  SIGMA_CHECK_ARG(kind != SIGMA_DIRS_CROSS || !det,
                  "sigma_ss2d_scan_bwd_saved_det: kind CROSS has no deterministic build (under the deterministic switch CroMB trains "
                  "through the op-level _det kernels)");
  SIGMA_CHECK_ARG(kind != SIGMA_DIRS_CROSS || batch % 2 == 0, "sigma_ss2d_scan_bwd_saved: CROSS needs batch = 2·images (batch=%d)", batch);
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && D > 0 && D % 64 == 0 && R > 0, "sigma_ss2d_scan_bwd_saved: bad sizes (D=%d must be a multiple of 64)", D);
  SIGMA_CHECK_ARG(N == 4 || N == 16, "sigma_ss2d_scan_bwd_saved: d_state=%d unsupported (4, 16)", N);
  SIGMA_CHECK_ARG(Cp == sigma_ss2d_padded_cp(N, R), "sigma_ss2d_scan_bwd_saved: Cp=%d must equal sigma_ss2d_padded_cp(N=%d, R=%d)", Cp, N, R);
  SIGMA_CHECK_ARG(al16(xc) && al16(xdbl) && al16(dy) && al16(delta) && al16(dxc) && al16(ddelta) && al16(dxdbl), "sigma_ss2d_scan_bwd_saved: pointers must be 16-byte aligned");
  SIGMA_CHECK_ARG(al16(hs), "sigma_ss2d_scan_bwd_saved: hs must be 16-byte aligned");
  return ss2d_scan_bwd(kind, xc, xdbl, dtw, dtb, A, Ds, dy, delta, hs, dxc, ddelta, dxdbl, dA, dDs, ddtb, batch, H, W, D, N, R, Cp, ws, wsb,
                       nsplit, (cudaStream_t)stream, det, xdtype);
}

// backward after sigma_ss2d_scan_fwd_save: `delta` and `hs` are INPUTS (what that call wrote)
int sigma_ss2d_scan_bwd_saved(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A, const float *Ds,
                              const float *dy, const float *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl, float *dA,
                              float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                              size_t workspace_bytes, int nsplit, void *stream) {
  SIGMA_CHECK_ARG(hs != nullptr, "sigma_ss2d_scan_bwd_saved: null hs");
  return ss2d_bwd_entry(kind, xc, xdbl, dtw, dtb, A, Ds, dy, delta, hs, dxc, ddelta, dxdbl, dA, dDs, ddtb, batch, H, W, D, N, R, Cp,
                        workspace, workspace_bytes, nsplit, stream);
}

// backward after sigma_ss2d_scan_fwd_save_bf16 / _fp16 (dtype SIGMA_BF16 / SIGMA_F16): xc, dy and delta are 16-bit; dxc and every
// other output fp32
static int ss2d_bwd_saved_16bit(const char *fn, int dtype, int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb,
                                const float *A, const float *Ds, const void *dy, const void *delta, const float *hs, float *dxc,
                                float *ddelta, float *dxdbl, float *dA, float *dDs, float *ddtb, int batch, int H, int W, int D, int N,
                                int R, int Cp, void *workspace, size_t workspace_bytes, int nsplit, void *stream) {
  SIGMA_CHECK_ARG(hs != nullptr, "%s: null hs", fn);
  SIGMA_CHECK_ARG(nsplit >= 0, "%s: nsplit=%d < 0", fn, nsplit);
  if (N == 8) {
    set_error("%s: d_state=8 unsupported (4, 16)", fn);
    return SIGMA_EUNSUPPORTED;
  }
  return ss2d_bwd_entry(kind, (const float *)xc, xdbl, dtw, dtb, A, Ds, (const float *)dy, (const float *)delta, hs, dxc, ddelta, dxdbl,
                        dA, dDs, ddtb, batch, H, W, D, N, R, Cp, workspace, workspace_bytes, nsplit, stream, 0, dtype);
}

int sigma_ss2d_scan_bwd_saved_bf16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                   const float *Ds, const void *dy, const void *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl,
                                   float *dA, float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                                   size_t workspace_bytes, int nsplit, void *stream) {
  return ss2d_bwd_saved_16bit("sigma_ss2d_scan_bwd_saved_bf16", SIGMA_BF16, kind, xc, xdbl, dtw, dtb, A, Ds, dy, delta, hs, dxc, ddelta,
                              dxdbl, dA, dDs, ddtb, batch, H, W, D, N, R, Cp, workspace, workspace_bytes, nsplit, stream);
}

int sigma_ss2d_scan_bwd_saved_fp16(int kind, const void *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                   const float *Ds, const void *dy, const void *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl,
                                   float *dA, float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                                   size_t workspace_bytes, int nsplit, void *stream) {
  return ss2d_bwd_saved_16bit("sigma_ss2d_scan_bwd_saved_fp16", SIGMA_F16, kind, xc, xdbl, dtw, dtb, A, Ds, dy, delta, hs, dxc, ddelta,
                              dxdbl, dA, dDs, ddtb, batch, H, W, D, N, R, Cp, workspace, workspace_bytes, nsplit, stream);
}

// the deterministic build of sigma_ss2d_scan_bwd_saved (nsplit = 0: the library's choice)
int sigma_ss2d_scan_bwd_saved_det(int kind, const float *xc, const float *xdbl, const float *dtw, const float *dtb, const float *A,
                                  const float *Ds, const float *dy, const float *delta, const float *hs, float *dxc, float *ddelta, float *dxdbl,
                                  float *dA, float *dDs, float *ddtb, int batch, int H, int W, int D, int N, int R, int Cp, void *workspace,
                                  size_t workspace_bytes, int nsplit, void *stream) {
  SIGMA_CHECK_ARG(hs != nullptr, "sigma_ss2d_scan_bwd_saved_det: null hs");
  SIGMA_CHECK_ARG(nsplit >= 0, "sigma_ss2d_scan_bwd_saved_det: nsplit=%d < 0", nsplit);
  return ss2d_bwd_entry(kind, xc, xdbl, dtw, dtb, A, Ds, dy, delta, hs, dxc, ddelta, dxdbl, dA, dDs, ddtb, batch, H, W, D, N, R, Cp,
                        workspace, workspace_bytes, nsplit, stream, 1);
}

int sigma_upsample2x_norm_fwd(const float *x, const float *w, const float *b, float *y, int batch, int H, int W, int C,
                              float eps, void *stream) {
  SIGMA_CHECK_ARG(x && y && ((w && b) || (!w && !b)), "sigma_upsample2x_norm_fwd: null pointer (w and b may be NULL together)");
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0, "sigma_upsample2x_norm_fwd: bad sizes");
  SIGMA_CHECK_ARG(al16(x) && al16(w) && al16(b) && al16(y), "sigma_upsample2x_norm_fwd: pointers must be 16-byte aligned");
  if (!w) return upsample2x_norm_launch(x, nullptr, nullptr, nullptr, 0, y, batch, H, W, C, eps, (cudaStream_t)stream);
  return upsample2x_norm_launch(x, w, b, nullptr, 0, y, batch, H, W, C, eps, (cudaStream_t)stream);
}

int sigma_upsample2x_norm_head_fwd(const float *x, const float *w, const float *b, const float *wcls, int num_classes,
                                   float *logits, int batch, int H, int W, int C, float eps, void *stream) {
  SIGMA_CHECK_ARG(x && w && b && wcls && logits, "sigma_upsample2x_norm_head_fwd: null pointer");
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && C > 0 && C % 4 == 0 && num_classes > 0,
                  "sigma_upsample2x_norm_head_fwd: bad sizes");
  SIGMA_CHECK_ARG(al16(x) && al16(w) && al16(b) && al16(wcls), "sigma_upsample2x_norm_head_fwd: pointers must be 16-byte aligned");
  return upsample2x_norm_launch(x, w, b, wcls, num_classes, logits, batch, H, W, C, eps, (cudaStream_t)stream);
}

int sigma_argmax_hist_fwd(const float *logits, const void *labels, int label_bytes, uint64_t *hist, uint64_t *counts,
                          uint8_t *pred, int batch, int num_classes, int64_t HW, void *stream) {
  SIGMA_CHECK_ARG(logits && labels && hist && counts, "sigma_argmax_hist_fwd: null pointer");
  SIGMA_CHECK_ARG(batch > 0 && HW > 0 && num_classes > 0 && num_classes <= 238, "sigma_argmax_hist_fwd: bad sizes (1 <= classes <= 238: the per-CTA histogram lives in shared memory)");
  return argmax_hist_launch(logits, labels, label_bytes, (unsigned long long *)hist, (unsigned long long *)counts, pred, batch,
                            num_classes, HW, (cudaStream_t)stream);
}

int sigma_pool_avgmax_partial_fwd(const float *x, float *partial, int batch, int64_t L, int C, int nslice, void *stream) {
  SIGMA_CHECK_ARG(x && partial, "sigma_pool_avgmax_partial_fwd: null pointer");
  SIGMA_CHECK_ARG(batch > 0 && L > 0 && C > 0 && C % 4 == 0 && nslice > 0 && nslice <= 65535 && al16(x),
                  "sigma_pool_avgmax_partial_fwd: bad sizes / alignment");
  return pool_avgmax_partial_launch(x, partial, batch, L, C, nslice, (cudaStream_t)stream);
}

int sigma_scale_add_fwd(const float *a, const float *sa, const float *b, const float *sb, float *out, int64_t rows,
                        int64_t rows_per_batch, int C, void *stream) {
  SIGMA_CHECK_ARG(b && sb && out && (a == nullptr || sa != nullptr), "sigma_scale_add_fwd: null pointer");
  SIGMA_CHECK_ARG(rows >= 0 && rows_per_batch > 0 && C > 0 && C % 4 == 0 && al16(a) && al16(sa) && al16(b) && al16(sb) && al16(out),
                  "sigma_scale_add_fwd: bad sizes / alignment");
  return scale_add_launch(a, sa, b, sb, out, rows, rows_per_batch, C, (cudaStream_t)stream);
}

size_t sigma_scan_bwd_workspace_bytes(int batch, int dim, int seqlen, int dstate, int ngroups, int dtype) {
  if (dstate > 16) return scan_op_bwd_wide_workspace_bytes(batch, dim, seqlen, dstate, ngroups);   // 0 beyond 256
  const int eb = dtype == SIGMA_F32 ? 4 : 2;
  size_t w = align256(std::max(scan_op_bwd_workspace_bytes(batch, dim, seqlen, dstate, eb),
                               scan_op_bwd_tma_workspace_bytes(batch, dim, seqlen, std::min(dstate, 16), eb)));
  if (dtype != SIGMA_F32 && widen_shape_ok(dim, seqlen, dstate, ngroups, 2)) w += widen_bwd_bytes(batch, dim, seqlen, dstate, ngroups);
  return w;
}

// the deterministic build appends the partials of whichever kernel runs (TMA-staged or generic) to the workspace
size_t sigma_scan_bwd_det_workspace_bytes(int batch, int dim, int seqlen, int dstate, int ngroups, int dtype) {
  if (dstate > 16) return scan_op_bwd_wide_workspace_bytes(batch, dim, seqlen, dstate, ngroups);   // one kernel for both builds
  if (batch <= 0 || dim <= 0 || seqlen <= 0 || dstate <= 0 || dstate > 16 || ngroups <= 0 || dim % ngroups) return 0;
  return align256(sigma_scan_bwd_workspace_bytes(batch, dim, seqlen, dstate, ngroups, dtype)) +
         std::max(scan_op_bwd_tma_det_bytes(batch, dim, seqlen, dstate, ngroups), scan_op_bwd_det_bytes(batch, dim, seqlen, dstate, ngroups));
}

static int scan_bwd_entry(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                          const float *delta_bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                          float *dD, float *ddelta_bias, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                          int delta_softplus, void *workspace, size_t workspace_bytes, int force_split, cudaStream_t stream,
                          int det = 0) {
  SIGMA_CHECK_ARG(u && delta && A && B && C && dout && du && ddelta && dA && dB && dC, "sigma_scan_bwd: null pointer argument");
  SIGMA_CHECK_ARG((D == nullptr || dD != nullptr) && (delta_bias == nullptr || ddelta_bias != nullptr),
                  "sigma_scan_bwd: dD / ddelta_bias required when D / delta_bias are given");
  SIGMA_CHECK_ARG(batch > 0 && dim > 0 && seqlen > 0 && dstate > 0 && ngroups > 0 && dim % ngroups == 0,
                  "sigma_scan_bwd: bad sizes (batch=%d dim=%d seqlen=%d dstate=%d ngroups=%d)", batch, dim, seqlen, dstate, ngroups);
  SIGMA_CHECK_ARG(dtype == SIGMA_F32 || dtype == SIGMA_F16 || dtype == SIGMA_BF16, "sigma_scan_bwd: unknown dtype %d", dtype);
  if (dstate > 256) { set_error("sigma_scan_bwd: d_state=%d > 256 is not supported (selective_scan.cpp:290)", dstate); return SIGMA_EUNSUPPORTED; }
  const size_t need = det ? sigma_scan_bwd_det_workspace_bytes(batch, dim, seqlen, dstate, ngroups, dtype)
                          : sigma_scan_bwd_workspace_bytes(batch, dim, seqlen, dstate, ngroups, dtype);
  if (workspace == nullptr || workspace_bytes < need) {
    set_error("sigma_scan_bwd: needs %zu workspace bytes, got %zu", need, workspace_bytes);
    return SIGMA_EWORKSPACE;
  }
  if (dstate > 16) {   // one deterministic kernel for every entry point; nsplit has no effect (scan_op_bwd_wide.cu)
    if (dtype == SIGMA_F32)
      return scan_op_bwd_wide<float>(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim, seqlen,
                                     dstate, ngroups, delta_softplus, workspace, workspace_bytes, stream);
    if (dtype == SIGMA_F16)
      return scan_op_bwd_wide<__half>(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim,
                                      seqlen, dstate, ngroups, delta_softplus, workspace, workspace_bytes, stream);
    return scan_op_bwd_wide<__nv_bfloat16>(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim,
                                           seqlen, dstate, ngroups, delta_softplus, workspace, workspace_bytes, stream);
  }
  void *det_ws = nullptr;
  if (det) {   // the kernels see only the plain workspace; the partials follow it
    const size_t base = align256(sigma_scan_bwd_workspace_bytes(batch, dim, seqlen, dstate, ngroups, dtype));
    det_ws = (char *)workspace + base;
    workspace_bytes = base;
  }
  if (dtype == SIGMA_F32)
    return scan_bwd_dispatch<float>(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim,
                                    seqlen, dstate, ngroups, delta_softplus, workspace, workspace_bytes, force_split, stream, det_ws);
  if (dtype == SIGMA_F16)
    return scan_bwd_dispatch<__half>(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim,
                                     seqlen, dstate, ngroups, delta_softplus, workspace, workspace_bytes, force_split, stream, det_ws);
  return scan_bwd_dispatch<__nv_bfloat16>(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch,
                                          dim, seqlen, dstate, ngroups, delta_softplus, workspace, workspace_bytes, force_split,
                                          stream, det_ws);
}

int sigma_scan_bwd(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                   const float *delta_bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                   float *dD, float *ddelta_bias, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                   int delta_softplus, void *workspace, size_t workspace_bytes, void *stream_) {
  return scan_bwd_entry(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim, seqlen,
                        dstate, ngroups, dtype, delta_softplus, workspace, workspace_bytes, 0, (cudaStream_t)stream_);
}

// test hook: force the number of L-segments of the backward
int sigma_scan_bwd_split(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                         const float *delta_bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                         float *dD, float *ddelta_bias, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                         int delta_softplus, void *workspace, size_t workspace_bytes, int nsplit, void *stream_) {
  return scan_bwd_entry(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim, seqlen,
                        dstate, ngroups, dtype, delta_softplus, workspace, workspace_bytes, nsplit, (cudaStream_t)stream_);
}

int sigma_scan_bwd_det(const void *u, const void *delta, const float *A, const void *B, const void *C, const float *D,
                       const float *delta_bias, const void *dout, void *du, void *ddelta, float *dA, float *dB, float *dC,
                       float *dD, float *ddelta_bias, int batch, int dim, int seqlen, int dstate, int ngroups, int dtype,
                       int delta_softplus, void *workspace, size_t workspace_bytes, int nsplit, void *stream_) {
  SIGMA_CHECK_ARG(nsplit >= 0, "sigma_scan_bwd_det: nsplit=%d < 0", nsplit);
  return scan_bwd_entry(u, delta, A, B, C, D, delta_bias, dout, du, ddelta, dA, dB, dC, dD, ddelta_bias, batch, dim, seqlen,
                        dstate, ngroups, dtype, delta_softplus, workspace, workspace_bytes, nsplit, (cudaStream_t)stream_, 1);
}

int sigma_linear_tf32(const float *A, int64_t lda, const float *W, const float *bias, const float *residual, int64_t ldr,
                      const float *rscale, float *C, int64_t ldc, int64_t M, int N, int K, void *stream) {
  SIGMA_CHECK_ARG(A && W && C, "sigma_linear_tf32: null pointer");
  SIGMA_CHECK_ARG(M >= 0 && M < (1LL << 31) && N > 0 && K > 0, "sigma_linear_tf32: bad sizes M=%lld N=%d K=%d", (long long)M, N, K);
  SIGMA_CHECK_ARG(K % 4 == 0 && N % 4 == 0 && lda % 4 == 0 && ldc % 4 == 0 && (residual == nullptr || ldr % 4 == 0) && lda >= K && ldc >= N,
                  "sigma_linear_tf32: K, N, lda, ldc, ldr must be multiples of 4 floats (16-byte TMA boxes; the epilogue reads bias / "
                  "rscale / residual as float4)");
  SIGMA_CHECK_ARG(al16(A) && al16(W) && al16(C) && al16(bias) && al16(residual) && al16(rscale),
                  "sigma_linear_tf32: pointers must be 16-byte aligned");
  SIGMA_CHECK_ARG(rscale == nullptr || residual != nullptr, "sigma_linear_tf32: rscale without residual");
  return gemm_launch(GemmOp::TF32, A, lda, W, nullptr, nullptr, nullptr, bias, residual, ldr, rscale, C, ldc, 0, M, N, K,
                     (cudaStream_t)stream);
}

int sigma_linear_bf16(const void *A, int64_t lda, const void *W, const float *bias, const float *residual, int64_t ldr,
                      const float *rscale, void *C, int64_t ldc, int c_dtype, int64_t M, int N, int K, void *stream) {
  return linear_16bit("sigma_linear_bf16", SIGMA_BF16, A, lda, W, bias, residual, ldr, rscale, C, ldc, c_dtype, M, N, K, stream);
}

int sigma_linear_fp16(const void *A, int64_t lda, const void *W, const float *bias, const float *residual, int64_t ldr,
                      const float *rscale, void *C, int64_t ldc, int c_dtype, int64_t M, int N, int K, void *stream) {
  return linear_16bit("sigma_linear_fp16", SIGMA_F16, A, lda, W, bias, residual, ldr, rscale, C, ldc, c_dtype, M, N, K, stream);
}

int sigma_linear_fp8(const void *A, int64_t lda, const float *sa, const void *Wq, const float *sw, const float *bias, const float *residual,
                     int64_t ldr, const float *rscale, void *C, int64_t ldc, int c_dtype, int64_t M, int N, int K, void *stream) {
  SIGMA_CHECK_ARG(A && sa && Wq && sw && C, "sigma_linear_fp8: null pointer");
  SIGMA_CHECK_ARG(c_dtype == SIGMA_F32 || c_dtype == SIGMA_BF16, "sigma_linear_fp8: c_dtype %d (SIGMA_F32 or SIGMA_BF16)", c_dtype);
  SIGMA_CHECK_ARG(M >= 0 && M < (1LL << 31) && N > 0 && K > 0, "sigma_linear_fp8: bad sizes M=%lld N=%d K=%d", (long long)M, N, K);
  SIGMA_CHECK_ARG(K % 16 == 0 && lda % 16 == 0 && N % 4 == 0 && ldc % 4 == 0 && (residual == nullptr || ldr % 4 == 0) && lda >= K && ldc >= N,
                  "sigma_linear_fp8: K and lda must be multiples of 16 (16-byte e4m3 TMA rows); N, ldc, ldr multiples of 4");
  SIGMA_CHECK_ARG(al16(A) && al16(Wq) && al16(C) && al16(bias) && al16(residual) && al16(rscale) && al8(sw),
                  "sigma_linear_fp8: A, Wq, C, bias, residual, rscale must be 16-byte and sw 8-byte aligned");
  SIGMA_CHECK_ARG(rscale == nullptr || residual != nullptr, "sigma_linear_fp8: rscale without residual");
  return gemm_launch(GemmOp::E4M3, A, lda, Wq, nullptr, sa, sw, bias, residual, ldr, rscale, C, ldc, c_dtype == SIGMA_BF16, M, N, K,
                     (cudaStream_t)stream);
}

int sigma_quantize_e4m3_rows(const void *x, int x_dtype, int64_t ldx, void *q, int64_t ldq, float *scale, int64_t rows, int C, void *stream) {
  SIGMA_CHECK_ARG(x && q && scale, "sigma_quantize_e4m3_rows: null pointer");
  SIGMA_CHECK_ARG(x_dtype == SIGMA_F32 || x_dtype == SIGMA_BF16, "sigma_quantize_e4m3_rows: x_dtype %d (SIGMA_F32 or SIGMA_BF16)", x_dtype);
  SIGMA_CHECK_ARG(rows >= 0 && C > 0 && C % 4 == 0 && ldx >= C && ldq >= C && ldx % 4 == 0 && ldq % 4 == 0,
                  "sigma_quantize_e4m3_rows: C=%d, ldx, ldq must be multiples of 4 with ldx, ldq >= C", C);
  SIGMA_CHECK_ARG((x_dtype == SIGMA_F32 ? al16(x) : al8(x)) && ((uintptr_t)q & 3) == 0,
                  "sigma_quantize_e4m3_rows: x must be 16-byte (fp32) or 8-byte (bf16) and q 4-byte aligned");
  return quantize_e4m3_rows_launch(x, x_dtype == SIGMA_BF16, ldx, q, ldq, scale, rows, C, (cudaStream_t)stream);
}

static int linear_tf32x3(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias, const float *residual,
                         int64_t ldr, const float *rscale, float *C, int64_t ldc, int64_t M, int N, int K, void *stream, bool reg_epilogue) {
  SIGMA_CHECK_ARG(A && W_hi && W_lo && C, "sigma_linear_tf32x3: null pointer");
  SIGMA_CHECK_ARG(M >= 0 && M < (1LL << 31) && N > 0 && K > 0, "sigma_linear_tf32x3: bad sizes M=%lld N=%d K=%d", (long long)M, N, K);
  SIGMA_CHECK_ARG(K % 4 == 0 && N % 4 == 0 && lda % 4 == 0 && ldc % 4 == 0 && (residual == nullptr || ldr % 4 == 0) && lda >= K && ldc >= N,
                  "sigma_linear_tf32x3: K, N, lda, ldc, ldr must be multiples of 4 floats");
  SIGMA_CHECK_ARG(al16(A) && al16(W_hi) && al16(W_lo) && al16(C) && al16(bias) && al16(residual) && al16(rscale),
                  "sigma_linear_tf32x3: pointers must be 16-byte aligned");
  SIGMA_CHECK_ARG(rscale == nullptr || residual != nullptr, "sigma_linear_tf32x3: rscale without residual");
  return gemm_launch(GemmOp::TF32X3, A, lda, W_hi, W_lo, nullptr, nullptr, bias, residual, ldr, rscale, C, ldc, 0, M, N, K,
                     (cudaStream_t)stream, reg_epilogue);
}

int sigma_linear_tf32x3(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias, const float *residual,
                        int64_t ldr, const float *rscale, float *C, int64_t ldc, int64_t M, int N, int K, void *stream) {
  return linear_tf32x3(A, lda, W_hi, W_lo, bias, residual, ldr, rscale, C, ldc, M, N, K, stream, false);
}

int sigma_test_linear_tf32x3_regs(const float *A, int64_t lda, const float *W_hi, const float *W_lo, const float *bias,
                                  const float *residual, int64_t ldr, const float *rscale, float *C, int64_t ldc, int64_t M, int N,
                                  int K, void *stream) {
  return linear_tf32x3(A, lda, W_hi, W_lo, bias, residual, ldr, rscale, C, ldc, M, N, K, stream, true);
}

int sigma_conv3x3_tf32(const float *x, const float *w9, const float *w9_lo, const float *bias, int act, float *y, int batch, int H, int W,
                       int Cin, int Cout, void *stream) {
  SIGMA_CHECK_ARG(x && w9 && y, "sigma_conv3x3_tf32: null pointer");
  SIGMA_CHECK_ARG(batch >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && Cin % 4 == 0 && Cout % 4 == 0,
                  "sigma_conv3x3_tf32: bad sizes (Cin=%d, Cout=%d must be multiples of 4)", Cin, Cout);
  SIGMA_CHECK_ARG(act == 0 || act == 1, "sigma_conv3x3_tf32: act must be 0 (none) or 1 (GELU)");
  SIGMA_CHECK_ARG(al16(x) && al16(w9) && al16(w9_lo) && al16(bias) && al16(y), "sigma_conv3x3_tf32: pointers must be 16-byte aligned");
  return conv3x3_tf32_launch(x, w9, w9_lo, bias, act, y, batch, H, W, Cin, Cout, (cudaStream_t)stream);
}

int sigma_conv3x3_gelu_save_tf32(const float *x, const float *w9, const float *w9_lo, const float *bias, float *y, float *pre, int batch,
                                 int H, int W, int Cin, int Cout, void *stream) {
  SIGMA_CHECK_ARG(x && w9 && y && pre, "sigma_conv3x3_gelu_save_tf32: null pointer");
  SIGMA_CHECK_ARG(batch >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && Cin % 4 == 0 && Cout % 4 == 0,
                  "sigma_conv3x3_gelu_save_tf32: bad sizes (Cin=%d, Cout=%d must be multiples of 4)", Cin, Cout);
  SIGMA_CHECK_ARG(al16(x) && al16(w9) && al16(w9_lo) && al16(bias) && al16(y) && al16(pre),
                  "sigma_conv3x3_gelu_save_tf32: pointers must be 16-byte aligned");
  return conv3x3_tf32_launch(x, w9, w9_lo, bias, 1, y, batch, H, W, Cin, Cout, (cudaStream_t)stream, 1, pre);
}

int sigma_conv3x3_dgrad_tf32(const float *dy, const float *w9t, const float *w9t_lo, const float *gelu_pre, float *dx, int batch, int H,
                             int W, int Cin, int Cout, void *stream) {
  SIGMA_CHECK_ARG(dy && w9t && dx, "sigma_conv3x3_dgrad_tf32: null pointer");
  SIGMA_CHECK_ARG(batch >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && Cin % 4 == 0 && Cout % 4 == 0,
                  "sigma_conv3x3_dgrad_tf32: bad sizes (Cin=%d, Cout=%d must be multiples of 4)", Cin, Cout);
  SIGMA_CHECK_ARG(al16(dy) && al16(w9t) && al16(w9t_lo) && al16(gelu_pre) && al16(dx),
                  "sigma_conv3x3_dgrad_tf32: pointers must be 16-byte aligned");
  // the conv of dy (Cout channels in) to dx (Cin channels out)
  return conv3x3_tf32_launch(dy, w9t, w9t_lo, nullptr, 0, dx, batch, H, W, Cout, Cin, (cudaStream_t)stream, gelu_pre ? 2 : 0,
                             (float *)gelu_pre);
}

size_t sigma_conv3x3_wgrad_workspace_bytes(int batch, int H, int W, int Cin, int Cout) {
  if (batch <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0) return 0;
  return conv3x3_wgrad_workspace_bytes(batch, H, W, Cin, Cout);
}

int sigma_conv3x3_wgrad_tf32(const float *x, int gelu_x, const float *dy, float *dw, float *dbias, int batch, int H, int W, int Cin,
                             int Cout, int x3, void *workspace, size_t workspace_bytes, void *stream) {
  SIGMA_CHECK_ARG(x && dy && dw, "sigma_conv3x3_wgrad_tf32: null pointer");
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && Cin % 4 == 0 && Cout % 4 == 0,
                  "sigma_conv3x3_wgrad_tf32: bad sizes batch=%d H=%d W=%d Cin=%d Cout=%d (Cin, Cout must be multiples of 4)", batch, H,
                  W, Cin, Cout);
  SIGMA_CHECK_ARG((gelu_x == 0 || gelu_x == 1) && (x3 == 0 || x3 == 1), "sigma_conv3x3_wgrad_tf32: gelu_x and x3 must be 0 or 1");
  SIGMA_CHECK_ARG(al16(x) && al16(dy), "sigma_conv3x3_wgrad_tf32: x and dy must be 16-byte aligned");
  const size_t need = conv3x3_wgrad_workspace_bytes(batch, H, W, Cin, Cout);
  if (workspace == nullptr || !al16(workspace) || workspace_bytes < need) {
    set_error("sigma_conv3x3_wgrad_tf32: needs %zu 16-byte aligned workspace bytes, got %zu", need, workspace ? workspace_bytes : 0);
    return SIGMA_EWORKSPACE;
  }
  return conv3x3_wgrad_launch(x, gelu_x, dy, dw, dbias, batch, H, W, Cin, Cout, x3, workspace, (cudaStream_t)stream);
}

int sigma_test_conv3x3_wgrad_plan(int batch, int H, int W, int Cin, int Cout, int64_t *out4_host) {
  SIGMA_CHECK_ARG(out4_host && batch > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "sigma_test_conv3x3_wgrad_plan: bad arguments");
  long long out[4];
  conv3x3_wgrad_plan(batch, H, W, Cin, Cout, out);
  for (int i = 0; i < 4; ++i) out4_host[i] = out[i];
  return SIGMA_OK;
}

// a pitch is a multiple of 4 elements (16 bytes: TMA strides, cp.async chunks) and holds the row's channels
static bool pitch_ok(int pitch, int count) { return pitch >= count && pitch % 4 == 0; }

int sigma_conv3x3_pitched_tf32(const float *x, int x_pitch, const float *w9, int w9_pitch, const float *w9_lo, const float *bias, int act,
                               float *y, int y_pitch, int batch, int H, int W, int Cin, int Cout, void *stream) {
  SIGMA_CHECK_ARG(x && w9 && y, "sigma_conv3x3_pitched_tf32: null pointer");
  SIGMA_CHECK_ARG(batch >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && (act == 0 || act == 1),
                  "sigma_conv3x3_pitched_tf32: bad sizes batch=%d H=%d W=%d Cin=%d Cout=%d or act=%d", batch, H, W, Cin, Cout, act);
  SIGMA_CHECK_ARG(pitch_ok(x_pitch, Cin) && pitch_ok(w9_pitch, Cin) && pitch_ok(y_pitch, Cout),
                  "sigma_conv3x3_pitched_tf32: pitches (x %d, w9 %d, y %d) must be multiples of 4 and at least Cin=%d / Cout=%d", x_pitch,
                  w9_pitch, y_pitch, Cin, Cout);
  SIGMA_CHECK_ARG(al16(x) && al16(w9) && al16(w9_lo) && al16(bias) && al16(y),
                  "sigma_conv3x3_pitched_tf32: pointers must be 16-byte aligned");
  return conv3x3_pitched_launch(x, x_pitch, w9, w9_lo, w9_pitch, bias, act, y, y_pitch, batch, H, W, Cin, Cout, (cudaStream_t)stream);
}

int sigma_conv3x3_gelu_save_pitched_tf32(const float *x, int x_pitch, const float *w9, int w9_pitch, const float *w9_lo,
                                         const float *bias, float *y, float *pre, int y_pitch, int batch, int H, int W, int Cin, int Cout,
                                         void *stream) {
  SIGMA_CHECK_ARG(x && w9 && y && pre, "sigma_conv3x3_gelu_save_pitched_tf32: null pointer");
  SIGMA_CHECK_ARG(batch >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0,
                  "sigma_conv3x3_gelu_save_pitched_tf32: bad sizes batch=%d H=%d W=%d Cin=%d Cout=%d", batch, H, W, Cin, Cout);
  SIGMA_CHECK_ARG(pitch_ok(x_pitch, Cin) && pitch_ok(w9_pitch, Cin) && pitch_ok(y_pitch, Cout),
                  "sigma_conv3x3_gelu_save_pitched_tf32: pitches (x %d, w9 %d, y %d) must be multiples of 4 and at least Cin=%d / "
                  "Cout=%d", x_pitch, w9_pitch, y_pitch, Cin, Cout);
  SIGMA_CHECK_ARG(al16(x) && al16(w9) && al16(w9_lo) && al16(bias) && al16(y) && al16(pre),
                  "sigma_conv3x3_gelu_save_pitched_tf32: pointers must be 16-byte aligned");
  return conv3x3_pitched_launch(x, x_pitch, w9, w9_lo, w9_pitch, bias, 1, y, y_pitch, batch, H, W, Cin, Cout, (cudaStream_t)stream, 1,
                                pre);
}

int sigma_conv3x3_dgrad_pitched_tf32(const float *dy, int dy_pitch, const float *w9t, int w9t_pitch, const float *w9t_lo,
                                     const float *gelu_pre, float *dx, int dx_pitch, int batch, int H, int W, int Cin, int Cout,
                                     void *stream) {
  SIGMA_CHECK_ARG(dy && w9t && dx, "sigma_conv3x3_dgrad_pitched_tf32: null pointer");
  SIGMA_CHECK_ARG(batch >= 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0,
                  "sigma_conv3x3_dgrad_pitched_tf32: bad sizes batch=%d H=%d W=%d Cin=%d Cout=%d", batch, H, W, Cin, Cout);
  SIGMA_CHECK_ARG(pitch_ok(dy_pitch, Cout) && pitch_ok(w9t_pitch, Cout) && pitch_ok(dx_pitch, Cin),
                  "sigma_conv3x3_dgrad_pitched_tf32: pitches (dy %d, w9t %d, dx %d) must be multiples of 4 and at least Cout=%d / "
                  "Cin=%d", dy_pitch, w9t_pitch, dx_pitch, Cout, Cin);
  SIGMA_CHECK_ARG(al16(dy) && al16(w9t) && al16(w9t_lo) && al16(gelu_pre) && al16(dx),
                  "sigma_conv3x3_dgrad_pitched_tf32: pointers must be 16-byte aligned");
  // the conv of dy (Cout channels in) to dx (Cin channels out)
  return conv3x3_pitched_launch(dy, dy_pitch, w9t, w9t_lo, w9t_pitch, nullptr, 0, dx, dx_pitch, batch, H, W, Cout, Cin,
                                (cudaStream_t)stream, gelu_pre ? 2 : 0, (float *)gelu_pre);
}

int sigma_conv3x3_wgrad_pitched_tf32(const float *x, int x_pitch, int gelu_x, const float *dy, int dy_pitch, float *dw, float *dbias,
                                     int batch, int H, int W, int Cin, int Cout, int x3, void *workspace, size_t workspace_bytes,
                                     void *stream) {
  SIGMA_CHECK_ARG(x && dy && dw, "sigma_conv3x3_wgrad_pitched_tf32: null pointer");
  SIGMA_CHECK_ARG(batch > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0,
                  "sigma_conv3x3_wgrad_pitched_tf32: bad sizes batch=%d H=%d W=%d Cin=%d Cout=%d", batch, H, W, Cin, Cout);
  SIGMA_CHECK_ARG(pitch_ok(x_pitch, Cin) && pitch_ok(dy_pitch, Cout),
                  "sigma_conv3x3_wgrad_pitched_tf32: pitches (x %d, dy %d) must be multiples of 4 and at least Cin=%d / Cout=%d",
                  x_pitch, dy_pitch, Cin, Cout);
  SIGMA_CHECK_ARG((gelu_x == 0 || gelu_x == 1) && (x3 == 0 || x3 == 1),
                  "sigma_conv3x3_wgrad_pitched_tf32: gelu_x and x3 must be 0 or 1");
  SIGMA_CHECK_ARG(al16(x) && al16(dy), "sigma_conv3x3_wgrad_pitched_tf32: x and dy must be 16-byte aligned");
  const size_t need = conv3x3_wgrad_workspace_bytes(batch, H, W, Cin, Cout);
  if (workspace == nullptr || !al16(workspace) || workspace_bytes < need) {
    set_error("sigma_conv3x3_wgrad_pitched_tf32: needs %zu 16-byte aligned workspace bytes, got %zu", need,
              workspace ? workspace_bytes : 0);
    return SIGMA_EWORKSPACE;
  }
  return conv3x3_wgrad_launch(x, gelu_x, dy, dw, dbias, batch, H, W, Cin, Cout, x3, workspace, (cudaStream_t)stream, x_pitch, dy_pitch);
}

int sigma_split_tf32_fwd(const float *x, float *hi, float *lo, int64_t n, void *stream) {
  SIGMA_CHECK_ARG(x && hi && lo && n >= 0, "sigma_split_tf32_fwd: bad arguments");
  return split_tf32_launch(x, hi, lo, n, (cudaStream_t)stream);
}

int sigma_image_pre_fwd(const uint8_t *src, const uint8_t *labels, float *out, int64_t *labels_out, int H0, int W0, int SH, int SW,
                        double scale_y, double scale_x, int OH, int OW, int off_y, int off_x, int mirror_src, int mirror_out,
                        int label_pad, const int *clip4_host, const double *mean3, const double *std3, void *stream) {
  SIGMA_CHECK_ARG(src && out && mean3 && std3, "sigma_image_pre_fwd: null pointer");
  SIGMA_CHECK_ARG((labels == nullptr) == (labels_out == nullptr), "sigma_image_pre_fwd: labels and labels_out go together");
  SIGMA_CHECK_ARG(H0 > 0 && W0 > 0 && SH > 0 && SW > 0 && OH > 0 && OW > 0 && scale_y > 0 && scale_x > 0, "sigma_image_pre_fwd: bad sizes");
  ImagePreParams p;
  p.src = src; p.dst = out; p.lsrc = labels; p.ldst = (long long *)labels_out;
  p.H0 = H0; p.W0 = W0; p.SH = SH; p.SW = SW; p.OH = OH; p.OW = OW; p.off_y = off_y; p.off_x = off_x;
  p.mirror_src = mirror_src; p.mirror_out = mirror_out; p.label_pad = label_pad; p.scale_y = scale_y; p.scale_x = scale_x;
  p.clip_y0 = 0; p.clip_x0 = 0; p.clip_y1 = SH; p.clip_x1 = SW;
  if (clip4_host) {
    p.clip_y0 = std::max(0, clip4_host[0]); p.clip_x0 = std::max(0, clip4_host[1]);
    p.clip_y1 = std::min(SH, clip4_host[0] + clip4_host[2]); p.clip_x1 = std::min(SW, clip4_host[1] + clip4_host[3]);
  }
  for (int c = 0; c < 3; ++c) {
    SIGMA_CHECK_ARG(std3[c] != 0.0, "sigma_image_pre_fwd: std[%d] == 0", c);
    p.mean[c] = mean3[c]; p.stdv[c] = std3[c];
  }
  return image_pre_launch(p, (cudaStream_t)stream);
}

int sigma_eval_exp_accumulate_fwd(const float *logits, const float *logits_flip, float *acc, int ncls, int TH, int TW, int m_top,
                                  int m_left, int vh, int vw, int AH, int AW, int ay, int ax, void *stream) {
  SIGMA_CHECK_ARG(logits && acc, "sigma_eval_exp_accumulate_fwd: null pointer");
  SIGMA_CHECK_ARG(ncls > 0 && m_top >= 0 && m_left >= 0 && vh >= 0 && vw >= 0 && m_top + vh <= TH && m_left + vw <= TW && ay >= 0 &&
                      ax >= 0 && ay + vh <= AH && ax + vw <= AW,
                  "sigma_eval_exp_accumulate_fwd: window (%d+%d, %d+%d) of a %dx%d tile into (%d, %d) of %dx%d", m_top, vh, m_left, vw,
                  TH, TW, ay, ax, AH, AW);
  return eval_exp_accumulate_launch(logits, logits_flip, acc, ncls, TH, TW, m_top, m_left, vh, vw, AH, AW, ay, ax, (cudaStream_t)stream);
}

int sigma_eval_resize_add_fwd(const float *acc, int ncls, int AH, int AW, int m_top, int m_left, int SH, int SW, double *out, int H0,
                              int W0, void *stream) {
  SIGMA_CHECK_ARG(acc && out, "sigma_eval_resize_add_fwd: null pointer");
  SIGMA_CHECK_ARG(ncls > 0 && SH > 0 && SW > 0 && H0 > 0 && W0 > 0 && m_top >= 0 && m_left >= 0 && m_top + SH <= AH && m_left + SW <= AW,
                  "sigma_eval_resize_add_fwd: bad sizes");
  return eval_resize_add_launch(acc, ncls, AH, AW, m_top, m_left, SH, SW, out, H0, W0, (cudaStream_t)stream);
}

int sigma_eval_argmax_hist_fwd(const double *score, const uint8_t *labels, uint8_t *pred, uint64_t *hist, uint64_t *counts,
                               int num_classes, int64_t HW, void *stream) {
  SIGMA_CHECK_ARG(score && pred, "sigma_eval_argmax_hist_fwd: null pointer");
  SIGMA_CHECK_ARG(labels == nullptr || (hist && counts), "sigma_eval_argmax_hist_fwd: labels need hist and counts");
  SIGMA_CHECK_ARG(num_classes >= 1 && num_classes <= 255 && HW >= 0, "sigma_eval_argmax_hist_fwd: bad sizes");
  if (HW == 0) return SIGMA_OK;
  return eval_argmax_hist_launch(score, labels, pred, (unsigned long long *)hist, (unsigned long long *)counts, num_classes, HW,
                                 (cudaStream_t)stream);
}

#pragma GCC visibility pop
}  // extern "C"
