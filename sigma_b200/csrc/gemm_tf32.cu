// Dense projections of the hot path (in_proj / x_proj / out_proj / PatchMerging / PatchExpand / decoder linears,
// vmamba.py:679,195,725,616; MambaDecoder.py:17,39,82-83) as ONE hand-written sm_90a GEMM:
//
//     C[M,N] = A[M,K] · W[N,K]^T  (+ bias[N])  (+ residual[M,N] · rscale[N])      fp32 in / fp32 out
//
// Hopper warpgroup MMA: `wgmma.mma_async ... m64nBNk8.f32.tf32.tf32`, fp32 operands read as TF32 straight from shared
// memory (no conversion pass), fp32 accumulators in registers.  Operand tiles are staged by TMA (128-byte swizzle) through
// a full/empty mbarrier ring.  Warp roles (288 threads): warps 0-7 = two consumer warpgroups, each owning 64 rows of the
// 128 x BN tile (its own A half, all of W) and issuing the MMAs for them; warp 8 = TMA producer.  Persistent CTAs loop over
// 128 x BN output tiles (BN a multiple of 32 up to 256, one template instance per width, chosen per call); the producer
// runs ahead across tile boundaries, so the loads of the next tile overlap the epilogue of the current one.  The epilogue
// adds bias / residual·rscale to the register accumulators and stores them directly (each warp store covers 8 rows x 32 B);
// the tf32x3 linear instance (gemm_x3_tma_kernel) stages them in shared memory and stores them with TMA instead (GemmEpi::TMA).
// These GEMMs are HBM-bound at the Sigma shapes (K = 96..1536): what matters is one pass over A and one over C.
//
// GemmOp::TF32X3 (sigma_linear_tf32x3): fp32-grade products on the TF32 tensor pipe by error compensation,
//     A·W = A_hi·W_hi + A_lo·W_hi + A_hi·W_lo  (+ A_lo·W_lo ~ 2^-22, dropped),   x_hi = x with the low 13 mantissa bits cleared.
// GemmSrc::CONV (sigma_conv3x3_tf32): the SAME kernel as an implicit-GEMM 3x3 convolution (pad 1, stride 1) over a channels-last
// (B, H, W, Cin) tensor: an M tile is an 8 x 16 pixel patch, the K loop runs over 9 taps x Cin blocks, and the A tile of tap
// (dy, dx) is ONE 4-D TMA box of the input shifted by (dy-1, dx-1) whose out-of-bounds fill is the zero padding (no im2col
// tensor); weights are (9, Cout, Cin); bias and an optional exact GELU are fused in the epilogue.  Replaces the
// ChannelAttentionBlock's two dense convolutions (vmamba.py:1749-1752).
//
// W_hi / W_lo come pre-split from the caller (weights: split once, sigma_split_tf32_fwd) and are read by the MMAs from shared
// memory; the activations feed wgmma from registers: per k8 step each thread loads its A fragment from the stage with one
// ldmatrix, splits it in registers (hi = mask, lo = v - hi) and issues three MMAs.  hi is masked explicitly, so the products
// do not depend on whether the tensor core truncates or rounds its fp32 operands to TF32.
#include <stdlib.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "tma.cuh"

namespace sigma {

constexpr int GM_BM = 128;       // rows per CTA tile = two warpgroups x wgmma M (64)
constexpr int GM_BK = 32;        // fp32 elements per k-block = one 128-byte swizzle row
constexpr int GM_UK = 8;         // wgmma K for tf32 (32 bytes)
constexpr int GM_THREADS = 288;  // two consumer warpgroups + one producer warp

// The FP8 instance's widest tile.  acc and the k-block fragment take BN registers per thread, so only BN <= 64 fits two CTAs
// per SM (96 registers at 64; 96 and 128 wide tiles take 114 / 146 and run one CTA per SM, 160 spills).  On an H100 the
// 64-wide tiles at two CTAs per SM ran Sigma-tiny's quantized GEMMs 1.1-2.1x faster than 128-wide ones at one, whose
// epilogue stores nothing overlaps (DESIGN §5.4), so the instance has the widths 32 and 64 only.
constexpr int kFp8MaxBn = 64;
// The widest tile of the conv's training epilogues (conv3x3_epi_kernel, cab_conv_pitched_kernel's EPI 1 / 2): the CAB's C/3
// (32 / 64 / 128 in Sigma-tiny and -small) fits one tile; wider outputs (Sigma-base's 170) take several.  The training
// epilogues keep two CTAs per SM, whose register budget ends at 128-column tiles (plan_gemm).
constexpr int kEpiMaxBn = 128;

// What the body and the host take from the operand kind; the wgmma form is wgmma_ss<OP, BN> (tf32x3: wgmma_tf32_rs) and the
// 16-bit type of C is GemmC16<OP>
struct GemmOpTraits {
  int bytes;                 // per operand element: a k-block is one 128-byte swizzle row, GM_BK·4 / bytes elements
  int max_bn;                // the widest tile instance
  CUtensorMapDataType tma;   // the operand tensor maps' element type
};
__host__ __device__ constexpr GemmOpTraits gemm_op_traits(GemmOp op) {
  return op == GemmOp::E4M3   ? GemmOpTraits{1, kFp8MaxBn, CU_TENSOR_MAP_DATA_TYPE_UINT8}
         : op == GemmOp::BF16 ? GemmOpTraits{2, 256, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16}
         : op == GemmOp::F16  ? GemmOpTraits{2, 256, CU_TENSOR_MAP_DATA_TYPE_FLOAT16}
                              : GemmOpTraits{4, 256, CU_TENSOR_MAP_DATA_TYPE_FLOAT32};
}
// The type C is stored in when p.c_bf16 is set; float: the fp32 kinds store fp32 C only
template <GemmOp OP>
using GemmC16 = std::conditional_t<OP == GemmOp::F16, __half,
                                   std::conditional_t<OP == GemmOp::BF16 || OP == GemmOp::E4M3, __nv_bfloat16, float>>;

// Where the A tiles come from: rows of a matrix, or the taps of a 3x3 conv over a channels-last tensor whose rows are Cin
// (CONV) or a pitch (PITCHED) elements apart
enum class GemmSrc { ROWS, CONV, PITCHED };
// What the epilogue does with the accumulators: store C from registers (REGS; the conv's plain or GELU output), or through
// shared memory with TMA (TMA); the conv's training epilogues also store pre = conv + bias to p.aux (PRE), or multiply the
// result by GELU'(p.aux) (DGELU)
enum class GemmEpi { REGS, TMA, PRE, DGELU };
// The instances there are: every kind on rows with C stored from registers, tf32x3 on rows with the TMA-stored epilogue, and
// the fp32 kinds' convs with the conv epilogues
constexpr bool gemm_instance_ok(GemmOp op, GemmSrc src, GemmEpi epi) {
  return src == GemmSrc::ROWS ? epi == GemmEpi::REGS || (epi == GemmEpi::TMA && op == GemmOp::TF32X3)
                              : (op == GemmOp::TF32 || op == GemmOp::TF32X3) && epi != GemmEpi::TMA;
}

struct alignas(64) GemmParams {
  CUtensorMap m_a, m_w, m_wlo;
  const float *bias, *residual, *rscale;
  float *C;
  long long ldr, ldc;
  int M, N, K, BN, stages;   // BN: host-side choice of the template instance
  int c_bf16;       // 1 = C is stored as GemmC16 (bf16 or fp16; bias / residual / rscale stay fp32)
  int cH, cW, tiles_w, tiles_hw, kbc, act;   // CONV: image size, 8x16 patches per row / per image, Cin blocks per tap, activation
  const float *sa, *sw;   // E4M3: per-row scales of A, per-output-channel scales of W
  CUtensorMap m_c, m_r;   // GemmEpi::TMA: C and (if any) the residual, GM_CHUNK x 64 boxes
  float *aux;             // GemmEpi::PRE stores the pre-activation here, DGELU reads GELU's input from it (C's layout)
};

// One ring stage holds a k-block's K-major, 128-byte-swizzled operand tiles, each 1024-aligned: [A | W].  tf32x3 adds W_lo:
// the register-stored epilogue's stage is [A | W][A_lo | W_lo], whose A_lo tile nothing writes (A is split in registers), and
// the TMA-stored epilogue's is [A | W_hi | W_lo].  gemm_body's offsets and plan_gemm's sizes both come from here.
__host__ __device__ constexpr int gemm_w_bytes(int bn) { return (bn * GM_BK * 4 + 1023) & ~1023; }
__host__ __device__ constexpr int gemm_stage_bytes(int bn, bool x3, bool tma_c) {
  return tma_c ? GM_BM * GM_BK * 4 + 2 * gemm_w_bytes(bn) : (GM_BM * GM_BK * 4 + gemm_w_bytes(bn)) * (x3 ? 2 : 1);
}
// TMA-stored epilogue: each consumer warpgroup stages its 64 rows in chunks of GM_CHUNK columns (one 128-byte swizzle row per
// row, 8 KB) through two buffers after the ring
constexpr int GM_CHUNK = 32;
constexpr int GM_CHUNK_BYTES = 64 * GM_CHUNK * 4;
constexpr int GM_STAGING_BYTES = 2 * 2 * GM_CHUNK_BYTES;

constexpr int CV_TH = 8, CV_TW = 16;   // pixel patch of one M tile (8 x 16 = GM_BM)

// K-major, 128-byte-swizzled operand tile: rows are 128 B apart, 8-row groups 1024 B apart (SBO), layout type 1 =
// SWIZZLE_128B (sm_90 encoding).  Advancing along K inside the swizzle row = +32 B on the start address per wgmma K.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(const void *smem) {
  const uint32_t addr = smem_u32(smem);
  uint64_t d = 0;
  d |= (uint64_t)((addr >> 4) & 0x3FFF);          // start address, 16-byte units
  d |= (uint64_t)1 << 16;                          // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)(1024 >> 4) << 32;                // stride byte offset: 8 rows x 128 B
  d |= (uint64_t)1 << 62;                          // SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across an asynchronous MMA
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// four 8 x 4 fp32 matrices (8 rows of 16 bytes each, row addresses from lanes 8j..8j+7 for matrix j): r[j] of lane l = word
// l % 4 of row l / 4 of matrix j (a .b16 ldmatrix moves a 32-bit word as its two halves, in place)
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}

// The wgmma forms, one explicit specialisation per tile width N = 32 .. 256: D[64 x N] (+)= A[64 x k] · B[N x k]^T into N / 2
// fp32 accumulators per thread.  WG_ACC_<N> / WG_CON_<N> are the accumulators' asm placeholders and "+f" constraints, built
// from chunks of 8; WG_WIDTHS lists each width with the numbers of the six operands that can follow them (nvcc takes no named
// asm operands, so these are spelled out).  The host's kernel selection iterates the same table.
#define WG_P0 "%0, %1, %2, %3, %4, %5, %6, %7"
#define WG_P1 "%8, %9, %10, %11, %12, %13, %14, %15"
#define WG_P2 "%16, %17, %18, %19, %20, %21, %22, %23"
#define WG_P3 "%24, %25, %26, %27, %28, %29, %30, %31"
#define WG_P4 "%32, %33, %34, %35, %36, %37, %38, %39"
#define WG_P5 "%40, %41, %42, %43, %44, %45, %46, %47"
#define WG_P6 "%48, %49, %50, %51, %52, %53, %54, %55"
#define WG_P7 "%56, %57, %58, %59, %60, %61, %62, %63"
#define WG_P8 "%64, %65, %66, %67, %68, %69, %70, %71"
#define WG_P9 "%72, %73, %74, %75, %76, %77, %78, %79"
#define WG_P10 "%80, %81, %82, %83, %84, %85, %86, %87"
#define WG_P11 "%88, %89, %90, %91, %92, %93, %94, %95"
#define WG_P12 "%96, %97, %98, %99, %100, %101, %102, %103"
#define WG_P13 "%104, %105, %106, %107, %108, %109, %110, %111"
#define WG_P14 "%112, %113, %114, %115, %116, %117, %118, %119"
#define WG_P15 "%120, %121, %122, %123, %124, %125, %126, %127"
#define WG_ACC_32 WG_P0 ", " WG_P1
#define WG_ACC_64 WG_ACC_32 ", " WG_P2 ", " WG_P3
#define WG_ACC_96 WG_ACC_64 ", " WG_P4 ", " WG_P5
#define WG_ACC_128 WG_ACC_96 ", " WG_P6 ", " WG_P7
#define WG_ACC_160 WG_ACC_128 ", " WG_P8 ", " WG_P9
#define WG_ACC_192 WG_ACC_160 ", " WG_P10 ", " WG_P11
#define WG_ACC_224 WG_ACC_192 ", " WG_P12 ", " WG_P13
#define WG_ACC_256 WG_ACC_224 ", " WG_P14 ", " WG_P15
#define WG_D(c)                                                                                                                  \
  "+f"(d[8 * c]), "+f"(d[8 * c + 1]), "+f"(d[8 * c + 2]), "+f"(d[8 * c + 3]), "+f"(d[8 * c + 4]), "+f"(d[8 * c + 5]),            \
      "+f"(d[8 * c + 6]), "+f"(d[8 * c + 7])
#define WG_CON_32 WG_D(0), WG_D(1)
#define WG_CON_64 WG_CON_32, WG_D(2), WG_D(3)
#define WG_CON_96 WG_CON_64, WG_D(4), WG_D(5)
#define WG_CON_128 WG_CON_96, WG_D(6), WG_D(7)
#define WG_CON_160 WG_CON_128, WG_D(8), WG_D(9)
#define WG_CON_192 WG_CON_160, WG_D(10), WG_D(11)
#define WG_CON_224 WG_CON_192, WG_D(12), WG_D(13)
#define WG_CON_256 WG_CON_224, WG_D(14), WG_D(15)
// X(N, o0, .. o5): %o0 .. %o5 are the operands after the N / 2 accumulators
#define WG_WIDTHS(X)                 \
  X(32, 16, 17, 18, 19, 20, 21)      \
  X(64, 32, 33, 34, 35, 36, 37)      \
  X(96, 48, 49, 50, 51, 52, 53)      \
  X(128, 64, 65, 66, 67, 68, 69)     \
  X(160, 80, 81, 82, 83, 84, 85)     \
  X(192, 96, 97, 98, 99, 100, 101)   \
  X(224, 112, 113, 114, 115, 116, 117) \
  X(256, 128, 129, 130, 131, 132, 133)

// Both operands K-major in shared memory (descriptors da, db), every operand kind but tf32x3; scale_d = 0 overwrites D.  Each
// kind's k step (k8 tf32, k16 bf16 / fp16, k32 e4m3) is 32 bytes, so the swizzled stage layout and the +32 B descriptor advance
// are shared.  The 16-bit forms take the transpose flags (0: K-major); tf32 and e4m3 are K-major only.
template <GemmOp OP, int N>
__device__ __forceinline__ void wgmma_ss(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d);
#define WG_SS(OP, SHAPE, TAIL, N, a, b, s)                                                                                       \
  template <>                                                                                                                    \
  __device__ __forceinline__ void wgmma_ss<GemmOp::OP, N>(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {      \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #s ", 0;\n"                                                               \
                 "wgmma.mma_async.sync.aligned.m64n" #N SHAPE " {" WG_ACC_##N "}, %" #a ", %" #b ", p, 1, 1" TAIL ";\n}\n"       \
                 : WG_CON_##N                                                                                                    \
                 : "l"(da), "l"(db), "r"(scale_d));                                                                              \
  }
#define WG_SS_TF32(N, o0, o1, o2, ...) WG_SS(TF32, "k8.f32.tf32.tf32", "", N, o0, o1, o2)
#define WG_SS_BF16(N, o0, o1, o2, ...) WG_SS(BF16, "k16.f32.bf16.bf16", ", 0, 0", N, o0, o1, o2)
#define WG_SS_F16(N, o0, o1, o2, ...) WG_SS(F16, "k16.f32.f16.f16", ", 0, 0", N, o0, o1, o2)
#define WG_SS_E4M3(N, o0, o1, o2, ...) WG_SS(E4M3, "k32.f32.e4m3.e4m3", "", N, o0, o1, o2)
WG_WIDTHS(WG_SS_TF32)
WG_WIDTHS(WG_SS_BF16)
WG_WIDTHS(WG_SS_F16)
WG_WIDTHS(WG_SS_E4M3)

// D[64 x N] (+)= A[64 x 8] · B[N x 8]^T with A from registers (the .tf32 A fragment: a[0..3] = rows g, g + 8, g, g + 8 and
// columns t, t, t + 4, t + 4 of this warp's 16 rows, g = lane / 4, t = lane % 4) and B K-major in shared memory.  The a
// registers must not change until a wgmma.wait_group has retired the MMA that reads them.
template <int N>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d);
#define WG_RS(N, a0, a1, a2, a3, b, s)                                                                                           \
  template <>                                                                                                                    \
  __device__ __forceinline__ void wgmma_tf32_rs<N>(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {  \
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %" #s ", 0;\n"                                                               \
                 "wgmma.mma_async.sync.aligned.m64n" #N "k8.f32.tf32.tf32 {" WG_ACC_##N "}, {%" #a0 ", %" #a1 ", %" #a2      \
                 ", %" #a3 "}, %" #b ", p, 1, 1;\n}\n"                                                                          \
                 : WG_CON_##N                                                                                                    \
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));                                          \
  }
WG_WIDTHS(WG_RS)

// shared -> global, 2-D tile, bulk-group completion (SASS: UTMASTG); out-of-bounds elements are not written
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, const void *smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"((uint64_t)map),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}

// TMA_C: residual chunk number e of a warpgroup, columns col.. and rows row.. of the residual, into staging buffer e % 2
__device__ __forceinline__ void load_residual_chunk(const GemmParams &p, unsigned char *stg, uint64_t *rfull, uint32_t e, int col,
                                                    int row) {
  mbar_arrive_expect_tx(&rfull[e & 1], GM_CHUNK_BYTES);
  tma_load_2d(stg + (e & 1) * GM_CHUNK_BYTES, &p.m_r, &rfull[e & 1], col, row);
}

// d/du of nn.GELU()'s exact form u·Φ(u): Φ(u) + u·φ(u)
__device__ __forceinline__ float gelu_grad(float u) {
  return 0.5f * (1.f + erff(u * 0.70710678118654752f)) + u * 0.39894228040143268f * expf(-0.5f * u * u);
}

// The body of every instance, for the operand kind OP, the A source SRC and the epilogue EPI (gemm_instance_ok).
// E4M3 (gemm_fp8_kernel): 128 operands per k-block; each k-block's four k32 MMAs accumulate into a zeroed fragment that is
// then added to the fp32 accumulators in registers (the tensor core's e4m3 accumulation keeps fewer bits than fp32, DESIGN
// §5.4), and the epilogue scales acc[row, col] by sa[row]·sw[col] before the bias / residual.
// GemmEpi::TMA (gemm_x3_tma_kernel): the epilogue stages each warpgroup's output in GM_CHUNK-column chunks in shared memory and
// stores them with TMA, asynchronously, so the consumers go on to the next tile's MMAs while the stores drain; the residual
// chunks arrive by TMA as well, the first two during the tile's k-loop.
// PRE / DGELU (conv3x3_epi_kernel, the CAB convs' training instances): also store pre = conv + bias to p.aux before the GELU;
// multiply the result by GELU'(p.aux) (the data gradient of the second conv, emitted at the first conv's pre-activation).
// PITCHED (cab_conv_pitched_kernel): the conv's output rows (C and aux) are p.ldc elements apart instead of p.N, and N may be odd:
// an odd N's last column is loaded and stored alone.  The input's pitch is in its tensor map.
template <int BN, GemmOp OP, GemmSrc SRC = GemmSrc::ROWS, GemmEpi EPI = GemmEpi::REGS>
__device__ __forceinline__ void gemm_body(const GemmParams &p) {
  static_assert(gemm_instance_ok(OP, SRC, EPI), "no such instance");
  constexpr bool X3 = OP == GemmOp::TF32X3, FP8 = OP == GemmOp::E4M3;
  constexpr bool CONV = SRC != GemmSrc::ROWS, PITCHED = SRC == GemmSrc::PITCHED, TMA_C = EPI == GemmEpi::TMA;
  constexpr int KB = GM_BK * 4 / gemm_op_traits(OP).bytes;   // elements per k-block: one 128-byte swizzle row in every case
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const int S = p.stages;
  constexpr int a_bytes = GM_BM * GM_BK * 4, b_bytes = BN * GM_BK * 4;
  constexpr int a_half = a_bytes / 2;                                // one warpgroup's 64 rows
  constexpr int stage_bytes = gemm_stage_bytes(BN, X3, TMA_C);
  constexpr int wlo_off = TMA_C ? a_bytes + gemm_w_bytes(BN) : stage_bytes / 2 + a_bytes;   // X3: the W_lo tile in a stage
  uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + (size_t)S * stage_bytes + (TMA_C ? GM_STAGING_BYTES : 0));
  uint64_t *empty = full + S;
  uint64_t *rfull = empty + S;   // TMA_C: residual chunk loaded, one per staging buffer

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nkb = CONV ? 9 * p.kbc : (p.K + KB - 1) / KB;
  const int num_n = (p.N + BN - 1) / BN;
  const int num_m = CONV ? p.M : (p.M + GM_BM - 1) / GM_BM;      // CONV: p.M counts pixel patches
  const long long total = (long long)num_m * num_n;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.m_a);
    tma_prefetch_desc(&p.m_w);
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    if (TMA_C) for (int i = 0; i < 4; ++i) mbar_init(&rfull[i], 1);
    fence_mbar_init();
  }
  __syncthreads();

  // Persistent CTA: tiles blockIdx.x, +gridDim.x, ... (n fastest, so consecutive tiles re-read the same A rows from L2).
  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      long long it = 0;
      for (long long tile = blockIdx.x; tile < total; tile += gridDim.x) {
        const int m0 = (int)(tile / num_n) * GM_BM, n0 = (int)(tile % num_n) * BN;
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int st = (int)(it % S);
          mbar_wait_backoff(&empty[st], (uint32_t)(((it / S) & 1) ^ 1));
          unsigned char *sa = smem_raw + (size_t)st * stage_bytes;
          mbar_arrive_expect_tx(&full[st], (uint32_t)(a_bytes + (X3 ? 2 : 1) * b_bytes));
          if (CONV) {
            const int mt = (int)(tile / num_n);
            const int b = mt / p.tiles_hw, r = mt - b * p.tiles_hw, ty = r / p.tiles_w, tx = r - ty * p.tiles_w;
            const int tap = kb / p.kbc, kc = kb - tap * p.kbc, dy = tap / 3, dx = tap - 3 * dy;
            // the tap's input patch: shifted by (dy-1, dx-1); rows / columns outside the image arrive as zeros = the padding
            tma_load_4d(sa, &p.m_a, &full[st], kc * GM_BK, tx * CV_TW + dx - 1, ty * CV_TH + dy - 1, b);
            tma_load_2d(sa + a_bytes, &p.m_w, &full[st], kc * GM_BK, tap * p.N + n0);
            if (X3) tma_load_2d(sa + wlo_off, &p.m_wlo, &full[st], kc * GM_BK, tap * p.N + n0);
          } else {
            tma_load_2d(sa, &p.m_a, &full[st], kb * KB, m0);
            tma_load_2d(sa + a_bytes, &p.m_w, &full[st], kb * KB, n0);
            if (X3) tma_load_2d(sa + wlo_off, &p.m_wlo, &full[st], kb * GM_BK, n0);
          }
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups: wgmma (X3: A split in registers) -> epilogue =====
  const int wg = warp >> 2;                 // rows 64·wg .. +63 of the tile
  const int t = threadIdx.x & 127;
  // X3: this lane's ldmatrix row in its warpgroup's 64 x 32 A tile.  For k8 step k, matrix j = lane / 8 is (rows 16·(warp % 4)
  // + 8·(j & 1) .. +7, 16-byte chunk 2k + j / 2), so r[0..3] is the wgmma A fragment; SWIZZLE_128B stores chunk c of row r at
  // chunk c ^ (r % 8), which also puts the 8 rows of each matrix in distinct banks.
  const uint32_t a_lane = (uint32_t)(16 * (warp & 3) + 8 * ((lane >> 3) & 1) + (lane & 7)) * 128u + (uint32_t)(((lane >> 4) ^ (lane & 7)) << 4);
  long long it = 0;
  // TMA_C: this warpgroup's two staging buffers; chunk number e (counted over the CTA's tiles) uses buffer e % 2, whose
  // (e / 2)-th residual load completes phase (e / 2) % 2 of rfull[2·wg + e % 2].  Thread t = 0 issues and waits for the bulk
  // copies of the warpgroup.
  unsigned char *stg = smem_raw + (size_t)S * stage_bytes + wg * 2 * GM_CHUNK_BYTES;
  uint32_t ec = 0;
  // TMA_C: the warpgroup's 64 x BN block of a tile starts at row m0, column n0; nch of its chunks hold any of C (none when
  // its rows are past M)
  const auto block = [&](long long tile, int &m0, int &n0) {
    m0 = (int)(tile / num_n) * GM_BM + 64 * wg;
    n0 = (int)(tile % num_n) * BN;
    return m0 < p.M ? min(BN / GM_CHUNK, (p.N - n0 + GM_CHUNK - 1) / GM_CHUNK) : 0;
  };
  for (long long tile = blockIdx.x; tile < total; tile += gridDim.x) {
    if (TMA_C && p.residual && t == 0) {
      int m0, n0;
      const int nch = block(tile, m0, n0);
      tma_store_wait_read<0>();                 // the previous tile's stores have left both buffers
      for (int c = 0; c < min(nch, 2); ++c) load_residual_chunk(p, stg, &rfull[2 * wg], ec + c, n0 + GM_CHUNK * c, m0);
    }
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const int st = (int)(it % S);
      mbar_wait(&full[st], (uint32_t)((it / S) & 1));
      unsigned char *sa = smem_raw + (size_t)st * stage_bytes;
      if constexpr (X3) {
        // A from registers, W_hi / W_lo from shared memory.  Per k8 step, two commit groups, small terms first: {A_lo·W_hi}
        // and {A_hi·W_lo, A_hi·W_hi}.  Each group's fragment is loaded from the stage and split just before it is issued, after
        // a wait_group 1 has retired the group before the previous one, so at most 8 fragment registers are live (the
        // 2-CTA-per-SM widths have 96 registers for 64 accumulators) while one group is always queued.
        const uint32_t a_frag = smem_u32(sa + wg * a_half) + a_lane;
        const uint64_t db = wgmma_desc_sw128(sa + a_bytes), dbl = wgmma_desc_sw128(sa + wlo_off);
#pragma unroll
        for (int k = 0; k < GM_BK / GM_UK; ++k) {
          const uint32_t addr = a_frag ^ (uint32_t)(32 * k);   // the stage is 1024-aligned: bits 4-6 of a_frag are the row's XOR
          uint32_t lo[4], hi[4];
          ldmatrix_x4(lo, addr);
#pragma unroll
          for (int i = 0; i < 4; ++i)
            lo[i] = __float_as_uint(__uint_as_float(lo[i]) - __uint_as_float(lo[i] & 0xFFFFE000u));
          acc_fence(acc);
          wgmma_fence();
          wgmma_tf32_rs<BN>(acc, lo, db + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
          wgmma_commit();
          acc_fence(acc);
          wgmma_wait<1>();                          // the previous step's A_hi group
          // k = 0: that was the previous k-block's last group, so its stage is free now rather than one k-block later (the
          // ring is two stages deep at most X3 widths)
          if (k == 0 && prev >= 0 && t == 0) mbar_arrive(&empty[prev]);
          ldmatrix_x4(hi, addr);
#pragma unroll
          for (int i = 0; i < 4; ++i) hi[i] &= 0xFFFFE000u;
          acc_fence(acc);
          wgmma_fence();
          wgmma_tf32_rs<BN>(acc, hi, dbl + (uint64_t)(2 * k), 1u);
          wgmma_tf32_rs<BN>(acc, hi, db + (uint64_t)(2 * k), 1u);
          wgmma_commit();
          acc_fence(acc);
          wgmma_wait<1>();                          // this step's A_lo group
        }
      } else if constexpr (FP8) {
        const uint64_t da = wgmma_desc_sw128(sa + wg * a_half), db = wgmma_desc_sw128(sa + a_bytes);
        float part[BN / 2];
        acc_fence(part);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GM_BK / GM_UK; ++k)     // four k32 steps, +32 B each; the first one overwrites the fragment
          wgmma_ss<OP, BN>(part, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), k ? 1u : 0u);
        wgmma_commit();
        acc_fence(part);
        wgmma_wait<0>();                            // the k-block's MMAs are done: the stage is free, the fragment final
        acc_fence(part);
        if (t == 0) mbar_arrive(&empty[st]);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
        continue;
      } else {
        const uint64_t da = wgmma_desc_sw128(sa + wg * a_half), db = wgmma_desc_sw128(sa + a_bytes);
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GM_BK / GM_UK; ++k) {   // +32 B along K inside the swizzle row = +2 in 16-byte units
          wgmma_ss<OP, BN>(acc, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (kb | k) ? 1u : 0u);
        }
        wgmma_commit();
        acc_fence(acc);
        wgmma_wait<1>();                            // the MMAs of the previous k-block have read their stage
      }
      if (!X3 && prev >= 0 && t == 0) mbar_arrive(&empty[prev]);
      prev = st;
    }
    wgmma_wait<0>();
    acc_fence(acc);
    if (prev >= 0 && t == 0) mbar_arrive(&empty[prev]);

    if constexpr (TMA_C) {
      // per chunk: bias / residual·rscale added in registers (the register-stored epilogue's operations, in its order) into
      // the staging buffer in the C map's 128-byte-swizzled box layout, then one TMA store; TMA clips the M tail and the
      // columns past N.  The buffer a chunk writes was last stored from two chunks earlier: t = 0 waits for that store to be
      // read out before the warpgroup barrier that precedes the next chunk's writes (with a residual, before its reload).
      int m0, c_n0;
      const int nch = block(tile, m0, c_n0);
      const int rr = 16 * (warp & 3) + (lane >> 2);   // this lane's rows rr, rr + 8 of the block
#pragma unroll
      for (int c = 0; c < BN / GM_CHUNK; ++c) {
        if (c >= nch) break;
        const uint32_t e = ec + c;
        const uint32_t buf = smem_u32(stg) + (e & 1) * GM_CHUNK_BYTES;
        if (p.residual) mbar_wait(&rfull[2 * wg + (e & 1)], (e >> 1) & 1);
#pragma unroll
        for (int i = 0; i < GM_CHUNK / 8; ++i) {
          const int n = c_n0 + GM_CHUNK * c + 8 * i + 2 * (lane & 3);
          const bool in = n < p.N;                     // N is even, so a column pair is all-in or all-out
          const float2 b = p.bias && in ? __ldg(reinterpret_cast<const float2 *>(p.bias + n)) : make_float2(0.f, 0.f);
          const float2 sc = p.rscale && in ? __ldg(reinterpret_cast<const float2 *>(p.rscale + n)) : make_float2(0.f, 0.f);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = rr + 8 * h;
            const uint32_t q = buf + r * 128 + (((2 * i + ((lane & 3) >> 1)) ^ (r & 7)) << 4) + ((lane & 1) << 3);
            float2 o = make_float2(acc[4 * (GM_CHUNK / 8 * c + i) + 2 * h], acc[4 * (GM_CHUNK / 8 * c + i) + 2 * h + 1]);
            if (p.bias) { o.x += b.x; o.y += b.y; }
            if (p.residual) {
              float2 rv;
              asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(rv.x), "=f"(rv.y) : "r"(q) : "memory");
              if (p.rscale) { o.x = fmaf(rv.x, sc.x, o.x); o.y = fmaf(rv.y, sc.y, o.y); }
              else { o.x += rv.x; o.y += rv.y; }
            }
            asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(q), "f"(o.x), "f"(o.y) : "memory");
          }
        }
        fence_proxy_async();
        if (t == 0) tma_store_wait_read<0>();
        asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
        if (t == 0) {
          tma_store_2d(&p.m_c, stg + (e & 1) * GM_CHUNK_BYTES, c_n0 + GM_CHUNK * c, m0);
          tma_store_commit();
          if (p.residual && c + 2 < nch) {
            tma_store_wait_read<0>();
            load_residual_chunk(p, stg, &rfull[2 * wg], e + 2, c_n0 + GM_CHUNK * (c + 2), m0);
          }
        }
      }
      ec += nch;
      continue;
    }

    // epilogue: accumulator fragment (m64nBN, f32): acc[4i + 2h + j] = row 16·(warp % 4) + lane / 4 + 8h,
    // column 8i + 2·(lane % 4) + j of this warpgroup's 64 x BN block
    const int mt = (int)(tile / num_n), n0 = (int)(tile % num_n) * BN;
    int cb = 0, cy0 = 0, cx0 = 0;
    if (CONV) {
      cb = mt / p.tiles_hw;
      const int r = mt - cb * p.tiles_hw, ty = r / p.tiles_w;
      cy0 = ty * CV_TH; cx0 = (r - ty * p.tiles_w) * CV_TW;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = 64 * wg + 16 * (warp & 3) + (lane >> 2) + 8 * h;   // row inside the 128-row tile
      long long coff;   // element offset of the row in C (fp32 or, p.c_bf16, GemmC16)
      const float *rrow = nullptr;
      float srow = 1.f;   // E4M3: the activation row's scale
      if (CONV) {   // row r = pixel (r / 16, r % 16) of the 8 x 16 patch
        const int y = cy0 + r / CV_TW, x = cx0 + (r % CV_TW);
        if (y >= p.cH || x >= p.cW) continue;
        if constexpr (PITCHED) coff = (((long long)cb * p.cH + y) * p.cW + x) * p.ldc;
        else coff = (((long long)cb * p.cH + y) * p.cW + x) * p.N;
      } else {
        const int row = mt * GM_BM + r;
        if (row >= p.M) continue;
        coff = (long long)row * p.ldc;
        if (p.residual) rrow = p.residual + (long long)row * p.ldr;
        if constexpr (FP8) srow = __ldg(p.sa + row);
      }
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int n = n0 + 8 * i + 2 * (lane & 3);
        if (n >= p.N) continue;                        // N is even, so a column pair is all-in or all-out
        float2 o = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
        if constexpr (FP8) {
          const float2 sw = __ldg(reinterpret_cast<const float2 *>(p.sw + n));
          o.x = o.x * srow * sw.x; o.y = o.y * srow * sw.y;
        }
        if constexpr (PITCHED) {   // PITCHED: N may be odd, and column N - 1 of an odd N is the pair's only column
          if (n + 1 == p.N) {
            float v = o.x;
            if (p.bias) v += __ldg(p.bias + n);
            if constexpr (EPI == GemmEpi::PRE) p.aux[coff + n] = v;
            if constexpr (EPI == GemmEpi::DGELU) v *= gelu_grad(p.aux[coff + n]);
            if (p.act == 1) v = 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
            p.C[coff + n] = v;
            continue;
          }
        }
        if (p.bias) {
          const float2 b = __ldg(reinterpret_cast<const float2 *>(p.bias + n));
          o.x += b.x; o.y += b.y;
        }
        if (rrow) {
          const float2 rv = __ldg(reinterpret_cast<const float2 *>(rrow + n));
          if (p.rscale) {
            const float2 sc = __ldg(reinterpret_cast<const float2 *>(p.rscale + n));
            o.x = fmaf(rv.x, sc.x, o.x); o.y = fmaf(rv.y, sc.y, o.y);
          } else {
            o.x += rv.x; o.y += rv.y;
          }
        }
        if constexpr (EPI == GemmEpi::PRE) *reinterpret_cast<float2 *>(p.aux + coff + n) = o;
        if constexpr (EPI == GemmEpi::DGELU) {
          const float2 u = *reinterpret_cast<const float2 *>(p.aux + coff + n);
          o.x *= gelu_grad(u.x); o.y *= gelu_grad(u.y);
        }
        if (CONV && p.act == 1) {   // nn.GELU() (exact, erf)
          o.x = 0.5f * o.x * (1.f + erff(o.x * 0.70710678118654752f));
          o.y = 0.5f * o.y * (1.f + erff(o.y * 0.70710678118654752f));
        }
        if (std::is_same<GemmC16<OP>, __half>::value && p.c_bf16)
          *reinterpret_cast<__half2 *>(reinterpret_cast<__half *>(p.C) + coff + n) = __floats2half2_rn(o.x, o.y);
        else if (std::is_same<GemmC16<OP>, __nv_bfloat16>::value && p.c_bf16)
          *reinterpret_cast<__nv_bfloat162 *>(reinterpret_cast<__nv_bfloat16 *>(p.C) + coff + n) = __floats2bfloat162_rn(o.x, o.y);
        else
          *reinterpret_cast<float2 *>(p.C + coff + n) = o;
      }
    }
  }
  if (TMA_C && t == 0) tma_store_wait_all<0>();   // the shared memory the stores read stays until they are done
}

template <int BN, bool X3, bool CONV, bool BF16 = false>
__global__ void __launch_bounds__(GM_THREADS, BN <= 128 ? 2 : 1) gemm_tf32_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<BN, BF16 ? GemmOp::BF16 : X3 ? GemmOp::TF32X3 : GemmOp::TF32, CONV ? GemmSrc::CONV : GemmSrc::ROWS>(p);
}

// the conv wrappers' EPI: 0 = plain or (p.act) GELU, 1 = PRE, 2 = DGELU
constexpr GemmEpi conv_epi(int epi) { return epi == 1 ? GemmEpi::PRE : epi == 2 ? GemmEpi::DGELU : GemmEpi::REGS; }

// The conv's training instances (CabConvFn): EPI 1 = the forward that keeps the pre-activation, EPI 2 = the data gradient with the
// GELU' factor.  A separate kernel, so that gemm_tf32_kernel keeps its code; widths up to kEpiMaxBn.
template <int BN, bool X3, int EPI>
__global__ void __launch_bounds__(GM_THREADS, BN <= 128 ? 2 : 1) conv3x3_epi_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<BN, X3 ? GemmOp::TF32X3 : GemmOp::TF32, GemmSrc::CONV, conv_epi(EPI)>(p);
}

// The pitched conv (the CAB convs of Sigma-base, whose C/3 is not a multiple of 4): x, y and the weights have row pitches that are
// multiples of 4 elements while the channel counts need not be.  The tensor maps' widths are the logical counts, so TMA fills
// channels past them with zeros whatever the pad bytes hold; the epilogue addresses rows at p.ldc and never stores a column
// >= N.  EPI as conv3x3_epi_kernel's, and 0 = plain or (p.act) GELU.  Widths up to 256 for EPI 0, kEpiMaxBn for EPI 1 and 2.
template <int BN, bool X3, int EPI>
__global__ void __launch_bounds__(GM_THREADS, BN <= 128 ? 2 : 1) cab_conv_pitched_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<BN, X3 ? GemmOp::TF32X3 : GemmOp::TF32, GemmSrc::PITCHED, conv_epi(EPI)>(p);
}

// The tf32x3 linear instance with the TMA-stored epilogue: fp32 C (and residual) whose rows a tensor map can describe.
// Widths up to 96 run two CTAs per SM; from 128 on, the staging buffers leave room for one (plan_gemm) and its registers.
template <int BN>
__global__ void __launch_bounds__(GM_THREADS, BN < 128 ? 2 : 1) gemm_x3_tma_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<BN, GemmOp::TF32X3, GemmSrc::ROWS, GemmEpi::TMA>(p);
}

// The FP8 instance.  Its two accumulator sets (acc and the k-block fragment) need BN registers per thread; at BN <= kFp8MaxBn
// two CTAs per SM (<= 112 registers each) hold them without spilling.
template <int BN>
__global__ void __launch_bounds__(GM_THREADS, 2) gemm_fp8_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<BN, GemmOp::E4M3>(p);
}

// The fp16 instance: the bf16 instance's widths, ring and occupancy with `k16.f32.f16.f16` MMAs (a separate kernel, so that
// gemm_tf32_kernel<..., BF16> stays as it was)
template <int BN>
__global__ void __launch_bounds__(GM_THREADS, BN <= 128 ? 2 : 1) gemm_fp16_kernel(const __grid_constant__ GemmParams p) {
  gemm_body<BN, GemmOp::F16>(p);
}

// ---- host ----
// K-major operand map of kind op: 128-byte box rows (GM_BK·4 / bytes elements) with the 128-byte swizzle
static int make_tmap_2d_sw128(CUtensorMap *map, GemmOp op, const void *base, long long rows, long long cols, long long ld,
                              int box_rows) {
  const GemmOpTraits t = gemm_op_traits(op);
  const uint64_t dims[2] = {(uint64_t)cols, (uint64_t)rows}, str[1] = {(uint64_t)ld * t.bytes};
  const uint32_t box[2] = {(uint32_t)(GM_BK * 4 / t.bytes), (uint32_t)box_rows};
  return make_tmap(map, t.tma, 2, base, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
}

// BN is a multiple of 32 (one wgmma width per template instance); a last column tile that overhangs N is zero-filled by
// TMA on the W load and masked in the epilogue.
// With many row tiles (the throughput regime) this is the widest divisor of N (the A tile is re-read once per column tile);
// with few (small batch: M of a few hundred rows) narrower tiles put more CTAs to work: cost = waves over the persistent
// CTAs (one per SM) x (bn + 128), the shared-memory bytes an MMA k-step reads for a 128 x bn tile.
static int pick_bn(int N, long long m_tiles = 1 << 30, int max_bn = 256) {
  const int full = N <= max_bn ? ((N + 31) / 32) * 32 : max_bn;
  int best_bn = full;
  long long best = -1;
  for (int bn = full; bn >= 64; bn -= 32) {
    const long long tiles = m_tiles * ((N + bn - 1) / bn);    // a last column tile that overhangs N costs a full tile
    const long long cost = ((tiles + kNumSMs - 1) / kNumSMs) * (bn + 128);
    if (best < 0 || cost < best || (cost == best && N % bn == 0 && N % best_bn != 0)) { best = cost; best_bn = bn; }
  }
  return best_bn;
}

int gemm_pick_bn_hook(int N, long long m_tiles) { return pick_bn(N, m_tiles); }

// x -> (hi = x with the low 13 mantissa bits cleared, lo = x - hi): the operand split of the tf32x3 GEMM, for the weights
__global__ void split_tf32_kernel(const float *__restrict__ x, float *__restrict__ hi, float *__restrict__ lo, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    hi[i] = h;
    lo[i] = v - h;
  }
}

int split_tf32_launch(const float *x, float *hi, float *lo, long long n, cudaStream_t stream) {
  if (n == 0) return SIGMA_OK;
  split_tf32_kernel<<<(unsigned)std::min<long long>((n + 255) / 256, kNumSMs * 8), 256, 0, stream>>>(x, hi, lo, n);
  SIGMA_CHECK_LAUNCH();
  return SIGMA_OK;
}

// The launch plan of one call: tile width, ring depth, shared memory and persistent grid.  gemm_launch,
// conv3x3_launch and the sigma_test_gemm_plan hook all take it from plan_gemm, so a test that asserts a property of
// the plan (e.g. "every CTA walks >= 3 tiles") asserts it of the launch.
struct GemmPlan {
  int BN, stages, ctas_per_sm;
  unsigned grid;        // persistent CTAs
  long long tiles;      // 128 x BN output tiles
  size_t smem;          // dynamic shared memory per CTA
};

// SIGMA_GEMM_BN=<w> forces the tile width (a multiple of 32 in [32, 256]; anything else is an error, not clamped), read per
// call so that a test can run one shape at every width.  Returns 0 when unset, the width, or SIGMA_EINVAL.
static int forced_bn() {
  const char *e = getenv("SIGMA_GEMM_BN");
  if (e == nullptr || e[0] == '\0') return 0;
  char *end = nullptr;
  const long v = strtol(e, &end, 10);
  if (*end != '\0' || v < 32 || v > 256 || v % 32 != 0) {
    set_error("SIGMA_GEMM_BN=\"%s\": the GEMM tile width must be a multiple of 32 in [32, 256]", e);
    return SIGMA_EINVAL;
  }
  return (int)v;
}

// conv_B > 0: the implicit-GEMM 3x3 convolution of a (conv_B, conv_H, conv_W, K) input with N output channels (M unused).
// The widest tile is the kind's (E4M3: kFp8MaxBn, two CTAs per SM), and kEpiMaxBn for the conv's training epilogues.
// GemmEpi::TMA (the tf32x3 linear instance): the staging buffers come out of the budget before the ring.
static int plan_gemm(GemmOp op, GemmEpi epi, long long M, int N, int conv_B, int conv_H, int conv_W, GemmPlan *pl) {
  const bool conv = conv_B > 0, fp8 = op == GemmOp::E4M3, tma_c = epi == GemmEpi::TMA;
  const int max_bn = epi == GemmEpi::PRE || epi == GemmEpi::DGELU ? kEpiMaxBn : gemm_op_traits(op).max_bn;
  const long long m_tiles = conv ? (long long)conv_B * ((conv_W + CV_TW - 1) / CV_TW) * ((conv_H + CV_TH - 1) / CV_TH)
                                 : (M + GM_BM - 1) / GM_BM;
  int bn = pick_bn(N, conv ? 1 << 30 : m_tiles, max_bn);
  const int fbn = forced_bn();
  if (fbn < 0) return fbn;
  if (fbn > max_bn) {
    set_error("SIGMA_GEMM_BN=%d: %s tiles are at most %d wide", fbn, fp8 ? "the e4m3 GEMM's" : "this conv's", max_bn);
    return SIGMA_EINVAL;
  }
  if (fbn > 0) bn = fbn;
  pl->BN = bn;
  pl->tiles = m_tiles * ((N + bn - 1) / bn);
  const int stage_bytes = gemm_stage_bytes(bn, op == GemmOp::TF32X3, tma_c), staging = tma_c ? GM_STAGING_BYTES : 0;
  // up to 227 KB per block; tiles of <= 128 columns keep the ring small enough for two CTAs per SM (their register budget)
  int regs_ctas = bn <= (fp8 ? 64 : 128) ? 2 : 1;
  const auto ring = [&](int ctas) { return ((ctas == 2 ? 112 * 1024 : 226 * 1024) - 1024 - staging) / stage_bytes; };
  // TMA-stored: where the staging and a two-stage ring no longer fit twice per SM, one CTA with a deeper ring
  if (tma_c && regs_ctas == 2 && 2 * (2 * stage_bytes + staging + 2048) > 228 * 1024) regs_ctas = 1;
  pl->stages = std::max(2, std::min(8, ring(regs_ctas)));
  pl->smem = (size_t)pl->stages * stage_bytes + staging + 1024 /*barriers*/;
  pl->ctas_per_sm = std::max(1, std::min(regs_ctas, (int)((228 * 1024) / (pl->smem + 1024))));
  pl->grid = (unsigned)std::min<long long>(pl->tiles, (long long)kNumSMs * pl->ctas_per_sm);
  return SIGMA_OK;
}

// api.cu test hook: out = {BN, stages, grid, tiles, smem bytes, CTAs per SM}.  mode: 0 = tf32, 1 = tf32x3 with the
// register-stored epilogue (the conv, and sigma_test_linear_tf32x3_regs), 2 = bf16 (the bf16 instance stages the same bytes per
// k-block as tf32 — 128-byte rows — so its plan is the tf32 plan), 4 = e4m3 (the same stage bytes too, narrower widths),
// 5 = tf32x3 with the TMA-stored epilogue (linear only), 7 = fp16 (the bf16 plan); 3 and 6 are not modes.  The K loop does not
// enter the plan.
int gemm_plan_hook(long long M, int N, int K, int mode, int conv_B, int conv_H, int conv_W, long long *out) {
  (void)K;
  static const GemmOp ops[8] = {GemmOp::TF32, GemmOp::TF32X3, GemmOp::BF16, GemmOp::TF32,
                                GemmOp::E4M3, GemmOp::TF32X3, GemmOp::TF32, GemmOp::F16};
  if (mode < 0 || mode > 7 || mode == 3 || mode == 6 || (mode >= 2 && conv_B > 0)) {
    set_error("gemm plan: mode %d (0 tf32, 1 tf32x3, 2 bf16, 4 e4m3, 5 tf32x3 TMA-stored, 7 fp16; only 0 and 1 have a conv)", mode);
    return SIGMA_EINVAL;
  }
  GemmPlan pl;
  const int rc = plan_gemm(ops[mode], mode == 5 ? GemmEpi::TMA : GemmEpi::REGS, M, N, conv_B, conv_H, conv_W, &pl);
  if (rc) return rc;
  out[0] = pl.BN; out[1] = pl.stages; out[2] = pl.grid; out[3] = pl.tiles; out[4] = (long long)pl.smem; out[5] = pl.ctas_per_sm;
  return SIGMA_OK;
}

// The instance of width BN for (op, src, epi), one of gemm_instance_ok's; nullptr past the widest tile of E4M3 or of the conv's
// training epilogues
template <int BN>
static const void *gemm_kernel(GemmOp op, GemmSrc src, GemmEpi epi) {
  const bool x3 = op == GemmOp::TF32X3;
  if (src == GemmSrc::ROWS) {
    switch (op) {
      case GemmOp::TF32: return (const void *)gemm_tf32_kernel<BN, false, false>;
      case GemmOp::TF32X3:
        return epi == GemmEpi::TMA ? (const void *)gemm_x3_tma_kernel<BN> : (const void *)gemm_tf32_kernel<BN, true, false>;
      case GemmOp::BF16: return (const void *)gemm_tf32_kernel<BN, false, false, true>;
      case GemmOp::F16: return (const void *)gemm_fp16_kernel<BN>;
      case GemmOp::E4M3:
        if constexpr (BN <= kFp8MaxBn) return (const void *)gemm_fp8_kernel<BN>;
        break;
    }
    return nullptr;
  }
  if (epi == GemmEpi::REGS) {
    if (src == GemmSrc::CONV) return x3 ? (const void *)gemm_tf32_kernel<BN, true, true> : (const void *)gemm_tf32_kernel<BN, false, true>;
    return x3 ? (const void *)cab_conv_pitched_kernel<BN, true, 0> : (const void *)cab_conv_pitched_kernel<BN, false, 0>;
  }
  if constexpr (BN <= kEpiMaxBn) {
    const bool pre = epi == GemmEpi::PRE;
    if (src == GemmSrc::CONV)
      return x3 ? (pre ? (const void *)conv3x3_epi_kernel<BN, true, 1> : (const void *)conv3x3_epi_kernel<BN, true, 2>)
                : (pre ? (const void *)conv3x3_epi_kernel<BN, false, 1> : (const void *)conv3x3_epi_kernel<BN, false, 2>);
    return x3 ? (pre ? (const void *)cab_conv_pitched_kernel<BN, true, 1> : (const void *)cab_conv_pitched_kernel<BN, true, 2>)
              : (pre ? (const void *)cab_conv_pitched_kernel<BN, false, 1> : (const void *)cab_conv_pitched_kernel<BN, false, 2>);
  }
  return nullptr;
}

// Launches the instance for (op, src, epi) at the plan's width on its persistent grid
static int gemm_run(GemmOp op, GemmSrc src, GemmEpi epi, GemmParams &p, const GemmPlan &pl, cudaStream_t stream) {
  const void *kern = nullptr;
  switch (pl.BN) {
#define GEMM_KERNEL_AT(N, ...) case N: kern = gemm_kernel<N>(op, src, epi); break;
    WG_WIDTHS(GEMM_KERNEL_AT)
#undef GEMM_KERNEL_AT
  }
  if (kern == nullptr) {
    set_error("gemm: no instance of width %d for this operand kind and epilogue", pl.BN);
    return SIGMA_EINVAL;
  }
  p.BN = pl.BN;
  p.stages = pl.stages;
  SIGMA_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
  void *args[] = {&p};
  SIGMA_CHECK_CUDA(cudaLaunchKernel(kern, dim3(pl.grid), dim3(GM_THREADS), args, pl.smem, stream));
  count_launch();
  return SIGMA_OK;
}

int gemm_launch(GemmOp op, const void *A, long long lda, const void *W, const void *W_lo, const float *sa, const float *sw,
                const float *bias, const float *residual, long long ldr, const float *rscale, void *C, long long ldc, int c_16,
                long long M, int N, int K, cudaStream_t stream, bool reg_epilogue) {
  if (M == 0) return SIGMA_OK;
  const bool x3 = op == GemmOp::TF32X3;
  const GemmEpi epi = x3 && !reg_epilogue ? GemmEpi::TMA : GemmEpi::REGS;
  GemmPlan pl;
  int rc;
  if ((rc = plan_gemm(op, epi, M, N, 0, 0, 0, &pl))) return rc;
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.bias = bias; p.residual = residual; p.rscale = rscale; p.C = (float *)C; p.ldr = ldr; p.ldc = ldc; p.c_bf16 = c_16;
  p.sa = sa; p.sw = sw;
  p.M = (int)M; p.N = N; p.K = K;
  if ((rc = make_tmap_2d_sw128(&p.m_a, op, A, M, K, lda, GM_BM))) return rc;
  if ((rc = make_tmap_2d_sw128(&p.m_w, op, W, N, K, K, pl.BN))) return rc;
  if (x3 && (rc = make_tmap_2d_sw128(&p.m_wlo, op, W_lo, N, K, K, pl.BN))) return rc;
  if (epi == GemmEpi::TMA) {
    const uint64_t dims[2] = {(uint64_t)N, (uint64_t)M}, str_c[1] = {(uint64_t)ldc * 4}, str_r[1] = {(uint64_t)ldr * 4};
    const uint32_t box[2] = {GM_CHUNK, 64};
    if ((rc = make_tmap(&p.m_c, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, C, dims, str_c, box, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B))) return rc;
    if (residual && (rc = make_tmap(&p.m_r, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, residual, dims, str_r, box,
                                    CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B))) return rc;
  }
  return gemm_run(op, GemmSrc::ROWS, epi, p, pl, stream);
}

// 3x3 convolution, pad 1, stride 1, channels-last: y (B,H,W,Cout) = conv(x (B,H,W,Cin), W9 (9, Cout, Cin)) + bias, optional GELU,
// with x, W9 and y (and aux) rows x_ld, w_ld and y_ld elements apart: the tensor maps' widths are Cin, so channels past Cin arrive
// as zeros; the epilogue never stores a column >= Cout.  W9_lo == nullptr: plain TF32; else tf32x3 with W9 = W9_hi.  epi 1
// (act 1): pre = conv + bias also stored to aux; epi 2 (act 0): the result times GELU'(aux).
static int conv3x3_launch(GemmSrc src, const float *x, long long x_ld, const float *W9, const float *W9_lo, long long w_ld,
                          const float *bias, int act, float *y, long long y_ld, int B, int H, int W, int Cin, int Cout,
                          cudaStream_t stream, int epi, float *aux) {
  if (B == 0) return SIGMA_OK;
  const GemmOp op = W9_lo ? GemmOp::TF32X3 : GemmOp::TF32;
  GemmPlan pl;
  int rc;
  if ((rc = plan_gemm(op, conv_epi(epi), 0, Cout, B, H, W, &pl))) return rc;
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.bias = bias; p.C = y; p.aux = aux; p.ldc = y_ld;
  p.N = Cout; p.K = Cin;
  p.cH = H; p.cW = W; p.act = act;
  p.tiles_w = (W + CV_TW - 1) / CV_TW;
  p.tiles_hw = p.tiles_w * ((H + CV_TH - 1) / CV_TH);
  p.M = B * p.tiles_hw;
  p.kbc = (Cin + GM_BK - 1) / GM_BK;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)x_ld * 4, (uint64_t)W * x_ld * 4, (uint64_t)H * W * x_ld * 4};
    uint32_t box[4] = {(uint32_t)GM_BK, (uint32_t)CV_TW, (uint32_t)CV_TH, 1};
    if ((rc = make_tmap(&p.m_a, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, x, dims, str, box, CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_128B))) return rc;
  }
  if ((rc = make_tmap_2d_sw128(&p.m_w, op, W9, 9LL * Cout, Cin, w_ld, pl.BN))) return rc;
  if (W9_lo && (rc = make_tmap_2d_sw128(&p.m_wlo, op, W9_lo, 9LL * Cout, Cin, w_ld, pl.BN))) return rc;
  return gemm_run(op, src, conv_epi(epi), p, pl, stream);
}

// the unpitched conv: rows Cin (x, W9) and Cout (y, aux) elements apart
int conv3x3_tf32_launch(const float *x, const float *W9, const float *W9_lo, const float *bias, int act, float *y, int B, int H, int W,
                        int Cin, int Cout, cudaStream_t stream, int epi, float *aux) {
  return conv3x3_launch(GemmSrc::CONV, x, Cin, W9, W9_lo, Cin, bias, act, y, Cout, B, H, W, Cin, Cout, stream, epi, aux);
}

// The same conv on pitched rows (cab_conv_pitched_kernel): x (B,H,W,x_ld) holds Cin channels, W9 (9·Cout, w_ld) Cin, y and aux
// (B,H,W,y_ld) Cout; the pitches are multiples of 4 and at least the counts, which need not be.  The plan is the unpitched conv's.
int conv3x3_pitched_launch(const float *x, long long x_ld, const float *W9, const float *W9_lo, long long w_ld, const float *bias, int act,
                           float *y, long long y_ld, int B, int H, int W, int Cin, int Cout, cudaStream_t stream, int epi, float *aux) {
  return conv3x3_launch(GemmSrc::PITCHED, x, x_ld, W9, W9_lo, w_ld, bias, act, y, y_ld, B, H, W, Cin, Cout, stream, epi, aux);
}

}  // namespace sigma
