// Shared device helpers and host-side error plumbing for libsigma_b200 (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "internal.cuh"

namespace sigma {

constexpr float kLog2e = 1.4426950408889634f;
constexpr int kNumSMs = 132;   // H100 SXM: grid sizes and the launch cost models assume this many SMs

// workspace carving: every sub-buffer starts on a 256-byte boundary
inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

#define SIGMA_CHECK_ARG(cond, ...)         \
  do {                                     \
    if (!(cond)) {                         \
      ::sigma::set_error(__VA_ARGS__);     \
      return SIGMA_EINVAL;                 \
    }                                      \
  } while (0)

#define SIGMA_CHECK_CUDA(expr)                                                            \
  do {                                                                                    \
    cudaError_t _e = (expr);                                                              \
    if (_e != cudaSuccess) {                                                              \
      ::sigma::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                         __LINE__);                                                       \
      return SIGMA_ECUDA;                                                                 \
    }                                                                                     \
  } while (0)

#define SIGMA_CHECK_LAUNCH()                      \
  do {                                            \
    ::sigma::count_launch();                      \
    SIGMA_CHECK_CUDA(cudaPeekAtLastError());      \
  } while (0)

// ---- element conversions: fp32 <-> {fp32, fp16, bf16}; widening is exact, narrowing rounds to nearest even ----
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
// two fp32 -> one 32-bit word holding two 16-bit T (a at the lower address)
template <typename T> __device__ __forceinline__ uint32_t from_f32x2(float a, float b);
template <> __device__ __forceinline__ uint32_t from_f32x2<__half>(float a, float b) {
  const __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<const uint32_t *>(&h);
}
template <> __device__ __forceinline__ uint32_t from_f32x2<__nv_bfloat16>(float a, float b) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t *>(&h);
}

// ---- 4-element fp32 / bf16 / fp16 accesses (a float4 or 8 bytes of bf16 / fp16) ----
__device__ __forceinline__ float4 bf16x4_to_f4(uint2 u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xFFFF0000u));
}
__device__ __forceinline__ float4 ld4(const float *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ float4 ld4(const __nv_bfloat16 *p) { return bf16x4_to_f4(*reinterpret_cast<const uint2 *>(p)); }
__device__ __forceinline__ float4 ld4g(const float *p) { return __ldg(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 ld4g(const __nv_bfloat16 *p) { return bf16x4_to_f4(__ldg(reinterpret_cast<const uint2 *>(p))); }
__device__ __forceinline__ float4 ld4cs(const float *p) { return __ldcs(reinterpret_cast<const float4 *>(p)); }
__device__ __forceinline__ float4 ld4cs(const __nv_bfloat16 *p) { return bf16x4_to_f4(__ldcs(reinterpret_cast<const uint2 *>(p))); }
__device__ __forceinline__ void st4(float *p, float4 v) { *reinterpret_cast<float4 *>(p) = v; }
__device__ __forceinline__ void st4(__nv_bfloat16 *p, float4 v) {
  *reinterpret_cast<uint2 *>(p) = make_uint2(from_f32x2<__nv_bfloat16>(v.x, v.y), from_f32x2<__nv_bfloat16>(v.z, v.w));
}
// the same for fp16 (the fp16 inference mode); a store past ±65504 gives ±inf, as torch's .half()
__device__ __forceinline__ float4 f16x4_to_f4(uint2 u) {
  const float2 a = __half22float2(*reinterpret_cast<const __half2 *>(&u.x)), b = __half22float2(*reinterpret_cast<const __half2 *>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ float4 ld4(const __half *p) { return f16x4_to_f4(*reinterpret_cast<const uint2 *>(p)); }
__device__ __forceinline__ float4 ld4g(const __half *p) { return f16x4_to_f4(__ldg(reinterpret_cast<const uint2 *>(p))); }
__device__ __forceinline__ float4 ld4cs(const __half *p) { return f16x4_to_f4(__ldcs(reinterpret_cast<const uint2 *>(p))); }
__device__ __forceinline__ void st4(__half *p, float4 v) {
  *reinterpret_cast<uint2 *>(p) = make_uint2(from_f32x2<__half>(v.x, v.y), from_f32x2<__half>(v.z, v.w));
}

// ---- e4m3 rows with one fp32 scale per row (the FP8 inference mode; the formula is stated in sigma_b200.h) ----
// Output-type tag of the row-wise kernels: `out` holds e4m3 bytes, RowNormParams::qscale one scale per row.
struct E4M3Rows {};
// 448 / amax, the factor that maps a row onto e4m3's finite range; amax = 0 -> 1 (the row quantizes to zeros, scale 1);
// clamped to FLT_MAX so that a row of tiny values cannot make it infinite
__device__ __forceinline__ float e4m3_inv_scale(float amax) {
  return amax == 0.f ? 1.f : fminf(__fdiv_rn(448.f, amax), 3.4028234663852886e38f);
}
__device__ __forceinline__ float e4m3_scale(float amax) { return amax == 0.f ? 1.f : __fdiv_rn(amax, 448.f); }
// four fp32 -> four e4m3 bytes of v·inv (x at the lowest address), round to nearest even, saturating to ±448
__device__ __forceinline__ uint32_t e4m3x4(float4 v, float inv) {
  uint16_t lo, hi;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(__fmul_rn(v.y, inv)), "f"(__fmul_rn(v.x, inv)));
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(__fmul_rn(v.w, inv)), "f"(__fmul_rn(v.z, inv)));
  return (uint32_t)lo | ((uint32_t)hi << 16);
}
__device__ __forceinline__ float amax4(float4 v) { return fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))); }

// ---- device math ----
__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ float lg2(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// F.softplus with the default threshold 20 (selective_scan_fwd_kernel.cuh:133,
// selective_scan_interface.py:107), branch-free and with ONE MUFU op so it schedules inside the scan's inner loop
// (the SFU is the scan's busiest unit):
//   softplus(x) = max(x,0) + log1p(z),  z = exp(-|x|) in (0,1],  log1p(z) = z·q(z)
// q = degree-8 Chebyshev interpolant of log1p(z)/z on [0,1]: relative error of log1p < 2.5e-7 over the whole range
// evaluated in fp32 (the earlier series / MUFU.LG2 split needed a second MUFU op and reached 1e-5 for z > 2^-6).
// For x > 20, z < 2.1e-9 and the sum rounds to x, which is exactly the reference's thresholded branch.
__device__ __forceinline__ float softplus20(float x) {
  const float z = ex2(-fabsf(x) * kLog2e);
  float q = 0.005126102361828089f;
  q = fmaf(q, z, -0.029074065387248993f);
  q = fmaf(q, z, 0.0775160863995552f);
  q = fmaf(q, z, -0.13602247834205627f);
  q = fmaf(q, z, 0.19076880812644958f);
  q = fmaf(q, z, -0.2483539879322052f);
  q = fmaf(q, z, 0.3331812024116516f);
  q = fmaf(q, z, -0.4999944567680359f);
  q = fmaf(q, z, 0.9999999403953552f);
  return fmaf(q, z, fmaxf(x, 0.f));
}

// ---- fp32 pair arithmetic.  Hopper has no packed fp32x2 FMA, so a pair is two scalar fma.rn / mul.rn: the same
// rounding per lane as the packed form.  The pair helpers keep the kernels' state-pair structure.
struct f2 { float x, y; };
__device__ __forceinline__ unsigned long long pack2(float a, float b) {
  unsigned long long r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ f2 unpack2(unsigned long long r) {
  f2 d;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(d.x), "=f"(d.y) : "l"(r));
  return d;
}
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return f2{__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)}; }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return f2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }

// softplus20 of two values at once.  Same arithmetic per element as softplus20.
__device__ __forceinline__ f2 softplus20x2(float x0, float x1) {
  const f2 z = f2{ex2(-fabsf(x0) * kLog2e), ex2(-fabsf(x1) * kLog2e)};
  f2 q = fma2(f2{0.005126102361828089f, 0.005126102361828089f}, z, f2{-0.029074065387248993f, -0.029074065387248993f});
  q = fma2(q, z, f2{0.0775160863995552f, 0.0775160863995552f});
  q = fma2(q, z, f2{-0.13602247834205627f, -0.13602247834205627f});
  q = fma2(q, z, f2{0.19076880812644958f, 0.19076880812644958f});
  q = fma2(q, z, f2{-0.2483539879322052f, -0.2483539879322052f});
  q = fma2(q, z, f2{0.3331812024116516f, 0.3331812024116516f});
  q = fma2(q, z, f2{-0.4999944567680359f, -0.4999944567680359f});
  q = fma2(q, z, f2{0.9999999403953552f, 0.9999999403953552f});
  return fma2(q, z, f2{fmaxf(x0, 0.f), fmaxf(x1, 0.f)});
}

__device__ __forceinline__ float silu(float x) { return __fdividef(x, 1.f + ex2(-x * kLog2e)); }

// ---- cp.async (LDGSTS) ----
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, int src_bytes) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem, int src_bytes) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N));
}

__device__ __forceinline__ float f4_get(const float4 &v, int i) {
  return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}

}  // namespace sigma
