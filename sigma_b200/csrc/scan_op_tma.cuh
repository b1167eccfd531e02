// Shared pieces of the TMA-staged op-level scan kernels (forward: scan_op_tma.cu, backward: scan_op_bwd_tma.cu).
//
// Layout at the op boundary is the reference's (selective_scan.cpp:165-249): u / delta / out (batch, dim, L) and
// B / C (batch, groups, N, L), L contiguous, element type T in {fp32, fp16, bf16}.  A tile is 64 BYTES of L per row
// (16 fp32 / 32 half positions): u / delta / dout tiles are TMA boxes {64 B, DT channels} landing in shared memory
// with the 64-byte swizzle, so that the thread that owns a channel (= a row) reads its positions as 16-byte chunks
// without bank conflicts; the tensor maps ask for 256-byte L2 promotion so DRAM sees 256-byte bursts per row, not 64.
// B / C arrive as [N][64 B] boxes and are transposed (and widened to fp32) by each warp into a private
// [position][B(N) | C(N)] fp32 tile — the row format of the fused kernel — so the recurrence reads 4 states of one
// position per broadcast LDS.128 and runs over state pairs (common.cuh: fma2 / mul2).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "scan_core.cuh"
#include "tma.cuh"

namespace sigma {

constexpr int OPT_ROW_BYTES = 64;   // bytes of L per tile row
constexpr int OPT_HS_POS = 16;      // the backward's state checkpoints: one every 16 positions

template <typename T> struct OpT;
template <> struct OpT<float> {
  static constexpr int LT = 16;
  static constexpr CUtensorMapDataType kType = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
};
template <> struct OpT<__half> {
  static constexpr int LT = 32;
  static constexpr CUtensorMapDataType kType = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
};
template <> struct OpT<__nv_bfloat16> {
  static constexpr int LT = 32;
  static constexpr CUtensorMapDataType kType = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
};

// byte offset of 16-byte chunk c of row r inside a 64-byte-row tile written by TMA with CU_TENSOR_MAP_SWIZZLE_64B
// (address bits [4,6) are XORed with bits [7,9); the tile base is 512-byte aligned)
__device__ __forceinline__ uint32_t sw64_off(int r, int c) { return (uint32_t)(r * OPT_ROW_BYTES + ((c ^ ((r >> 1) & 3)) << 4)); }

// G consecutive positions (group g of the tile) of this thread's row -> fp32 registers
template <typename T, int G>
__device__ __forceinline__ void load_group(const unsigned char *tile, int r, int g, float (&v)[G]) {
  if constexpr (sizeof(T) == 4) {
#pragma unroll
    for (int q = 0; q < G / 4; ++q) {
      const float4 t = *reinterpret_cast<const float4 *>(tile + sw64_off(r, g * (G / 4) + q));
      v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
  } else {
    if constexpr (G == 8) {
      const uint4 t = *reinterpret_cast<const uint4 *>(tile + sw64_off(r, g));
      const T *e = reinterpret_cast<const T *>(&t);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = to_f32(e[i]);
    } else {
      const uint2 t = *reinterpret_cast<const uint2 *>(tile + sw64_off(r, g >> 1) + ((g & 1) << 3));
      const T *e = reinterpret_cast<const T *>(&t);
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = to_f32(e[i]);
    }
  }
}

// the inverse: G fp32 values -> T, stored at the same (swizzled) place of a tile
template <typename T, int G>
__device__ __forceinline__ void store_group(unsigned char *tile, int r, int g, const float (&v)[G]) {
  if constexpr (sizeof(T) == 4) {
#pragma unroll
    for (int q = 0; q < G / 4; ++q)
      *reinterpret_cast<float4 *>(tile + sw64_off(r, g * (G / 4) + q)) = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  } else {
    if constexpr (G == 8) {
      uint4 t;
      t.x = from_f32x2<T>(v[0], v[1]); t.y = from_f32x2<T>(v[2], v[3]);
      t.z = from_f32x2<T>(v[4], v[5]); t.w = from_f32x2<T>(v[6], v[7]);
      *reinterpret_cast<uint4 *>(tile + sw64_off(r, g)) = t;
    } else {
      uint2 t;
      t.x = from_f32x2<T>(v[0], v[1]); t.y = from_f32x2<T>(v[2], v[3]);
      *reinterpret_cast<uint2 *>(tile + sw64_off(r, g >> 1) + ((g & 1) << 3)) = t;
    }
  }
}

// One warp: raw B and C tiles ([NP rows][64 B], unswizzled, element type T) -> fp32 [LT][PITCH] rows [B(NP) | C(NP) | pad].
// PITCH = 2·NP + 4 floats keeps rows 16-byte aligned and spreads the transposed stores over 8 banks.
template <typename T, int NP>
__device__ __forceinline__ void transpose_bc(const unsigned char *rawB, const unsigned char *rawC, float *bct, int lane) {
  constexpr int LT = OpT<T>::LT, PITCH = 2 * NP + 4;
  constexpr int LPR = 32 / LT;           // fp32: 2 state rows per pass; half: 1
#pragma unroll
  for (int j = 0; j < NP / LPR; ++j) {
    const int l = lane % LT, n = j * LPR + lane / LT;
    const float b = to_f32(*reinterpret_cast<const T *>(rawB + n * OPT_ROW_BYTES + l * sizeof(T)));
    const float c = to_f32(*reinterpret_cast<const T *>(rawC + n * OPT_ROW_BYTES + l * sizeof(T)));
    bct[l * PITCH + n] = b;
    bct[l * PITCH + NP + n] = c;
  }
}

}  // namespace sigma
