// The selective-scan recurrence as executed by one thread (shared by the op-level kernel and the
// fused channels-last SS2D kernel).
//
// Mapping (GPU-first, not the reference's CUB block-scan): the sequence is walked SERIALLY by the
// thread that owns (channel d, SPT consecutive states); LPC = Npad/SPT lanes cooperate on one
// channel.  The state h stays in registers for the whole walk, so each (d,l,n) element costs
// exactly one MUFU.EX2 + 4 FP32-pipe ops — the SFU, not HBM, is the binding unit for N=16
// (SURVEY.md §7) and any block-scan formulation adds >= 2 FP32 ops per element on top.
// Parallelism along L, when the batch cannot fill the SMs, comes from splitting L into segments
// (MODE_SUMMARY -> combine -> MODE_APPLY below), not from a scan inside the CTA.
//
// Semantics follow selective_scan_fwd_kernel.cuh:126-189 / selective_scan_interface.py:100-131:
//   a = exp2(delta'·A·log2e);  h = a·h + (delta'·u)·B;  y += C·h
#pragma once
#include "common.cuh"

namespace sigma {

enum ScanMode { MODE_SERIAL = 0, MODE_SUMMARY = 1, MODE_APPLY = 2 };

// One scan position for SPT states.  Bs/Cs: this thread's SPT coefficients at that position.
template <int SPT, bool WITH_Y>
__device__ __forceinline__ void scan_step(float (&h)[SPT], const float (&a2)[SPT], float dl, float u,
                                          const float (&Bs)[SPT], const float (&Cs)[SPT], float &y) {
  const float dlu = dl * u;
#pragma unroll
  for (int s = 0; s < SPT; ++s) {
    const float a = ex2(dl * a2[s]);
    h[s] = fmaf(a, h[s], dlu * Bs[s]);
    if (WITH_Y) y = fmaf(h[s], Cs[s], y);
  }
}

// Sum `v` over the LPC lanes that share a channel (lanes are contiguous, LPC a power of two).
template <int LPC>
__device__ __forceinline__ float channel_reduce(float v) {
#pragma unroll
  for (int o = LPC / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The dB / dC reduction of the backward kernels: sum v[0..NV) over the W lanes {lane ^ x : x < W} (W a power of two <= 32).
// Halving steps trade registers for lanes: after the step with offset OFF a lane keeps the half of the values selected by
// (lane & OFF); when one value is left the remaining offsets are plain butterflies.  Returns the sum of value index `which`
// (also returned) — every value index is held by W / NV lanes.
template <int NV, int OFF>
__device__ __forceinline__ float transpose_reduce(float (&v)[NV], int lane, int &which) {
  if constexpr (OFF == 0) {
    return v[0];
  } else if constexpr (NV > 1) {
    const bool up = (lane & OFF) != 0;
    float w[NV / 2];
#pragma unroll
    for (int j = 0; j < NV / 2; ++j) {
      const float send = up ? v[j] : v[j + NV / 2];
      const float keep = up ? v[j + NV / 2] : v[j];
      w[j] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
    }
    which = which * 2 + (up ? 1 : 0);
    return transpose_reduce<NV / 2, OFF / 2>(w, lane, which);
  } else {
    float w[1] = {v[0] + __shfl_xor_sync(0xffffffffu, v[0], OFF)};
    return transpose_reduce<1, OFF / 2>(w, lane, which);
  }
}

// delta' for a group of 4 consecutive positions, computed ONCE per channel and shared by its LPC
// lanes: lane q evaluates softplus for position(s) it owns, then the values are exchanged by
// shuffle.  raw[i] must be identical across the LPC lanes of a channel.
template <int LPC>
__device__ __forceinline__ void shared_softplus4(const float (&raw)[4], bool softplus, int lane,
                                                 float (&dl)[4]) {
  if (LPC == 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i) dl[i] = softplus ? softplus20(raw[i]) : raw[i];
  } else if (LPC == 2) {
    const int q = lane & 1;
    float m0 = q ? raw[2] : raw[0], m1 = q ? raw[3] : raw[1];
    if (softplus) { m0 = softplus20(m0); m1 = softplus20(m1); }
    const int base = lane & ~1;
    dl[0] = __shfl_sync(0xffffffffu, m0, base);
    dl[1] = __shfl_sync(0xffffffffu, m1, base);
    dl[2] = __shfl_sync(0xffffffffu, m0, base + 1);
    dl[3] = __shfl_sync(0xffffffffu, m1, base + 1);
  } else {
    const int q = lane & 3;  // lanes q>=4 of a wider group duplicate lanes 0..3
    float m = q == 0 ? raw[0] : (q == 1 ? raw[1] : (q == 2 ? raw[2] : raw[3]));
    if (softplus) m = softplus20(m);
    const int base = lane & ~(LPC - 1);
#pragma unroll
    for (int i = 0; i < 4; ++i) dl[i] = __shfl_sync(0xffffffffu, m, base + i);
  }
}

}  // namespace sigma
