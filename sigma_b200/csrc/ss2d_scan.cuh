// a4+a5 — fused multi-direction SS2D scan, channels-last (see include/sigma_b200.h: sigma_ss2d_scan_fwd).
//
// One launch does, for every direction k of an SS2D block:
//   CrossScan (index math: each direction is a walk over the SAME channels-last tensor, expressed as a
//   4-D TMA tensor map — row-major = tiles along L, column-major = tiles along H at fixed w, reversed =
//   the same tiles walked backwards) -> dt_proj (R-term dot product, W_dt row in registers) -> +bias ->
//   softplus -> selective scan (state in registers, one MUFU.EX2 per element) -> D skip -> store at the
//   POSITION the value belongs to (so CrossMerge's un-flip / un-transpose disappear).
//
// Mapping: one thread owns one channel (CPT = 1; the template keeps a 2-channel variant that shares the B / C reads
// and lost at every measured shape, not instantiated) with all N states in registers; a warp covers 32 consecutive
// channels, so every global / shared access of a warp is a 128-byte row and B / C / dt_r are broadcast shared reads.
// No shuffles.  The recurrence is written over state pairs (common.cuh: fma2 / mul2, scalar fp32 on Hopper): per
// (channel, position) and state pair 2 MUL + 2 MUFU.EX2 + 2 MUL + 2 FFMA + 2 FFMA.
// CTA = (channel tile DT, direction k [x L-segment], image b) = DT/32 warps, all computing.
// Tiles of LT scan positions are staged HBM -> shared by TMA (cp.async.bulk.tensor) through a ring whose depth the
// host chooses (no CTA-wide barrier in the loop): a "full" mbarrier per slot signals TMA completion; a per-slot
// arrival counter replaces the usual "empty" barrier — the warp whose arrival completes a round (the LAST warp to
// finish the tile) immediately requests the tile that reuses the slot, so nobody ever waits for a slot and a tile
// is requested depth-1 tiles ahead of its first use.  An earlier version had a dedicated producer warp (a fifth of
// the CTA's registers).  Waits on "full" are non-suspending spins (test_wait): a suspended try_wait costs a
// microsecond-scale wake-up.
// y goes straight from registers to HBM (a warp writes 32 consecutive channels of one position = one 128-byte row).
// Per group of G positions the delta' of the NEXT group is computed in the same basic block as the recurrence of
// the current one (software pipelining across tile boundaries: the only serial dependency is h = a·h + b).
#pragma once
#include "scan_core.cuh"
#include <type_traits>

#include "tma.cuh"

namespace sigma {

template <int N>
struct Ss2dCfg {
  static constexpr int G = N >= 16 ? 4 : 8;       // positions per software-pipelined group (measured: 8/16 lose at N=16, 16 loses at N=4)
  static constexpr int LT = N >= 16 ? 16 : 32;    // scan positions per tile (multiple of G; measured: 16 loses at N=4)
  static constexpr int MAX_NST = 8;               // TMA ring depth is chosen on the host (Ss2dParams::nst), up to this
  static constexpr int MAXW = 4;                  // warps per CTA
  static constexpr int CTAS = 3;                  // default resident 128-thread CTAs per SM the register budget is set for (168 regs)
};
// The kernel is built for two register budgets (`__launch_bounds__(128, CTAS)`): 3 -> 168 registers (12 warps per SM)
// and, for d_state 16, 4 -> 128 registers (16 warps; no spills inside the position loop).  The host picks per
// (d_state, padded dt_rank) from measurements (ss2d_scan_host.cu: ss2d_pick_ctas).
__host__ __device__ constexpr int ss2d_reg_cap(int ctas) { return (65536 / (ctas * 128)) / 8 * 8; }

struct alignas(64) Ss2dParams {
  CUtensorMap m_xc[4], m_dbl[4];
  const float *dtw, *dtb, *A, *Ds;
  float *y, *carry;
  // training forward (SAVE kernels): what the fused backward (ss2d_scan_bwd.cu) reads instead of recomputing it —
  // delta' = softplus(dt_proj) slabs (K, batch, Lseq, D), stored like y, and the state at the start of every 16-position block
  // of the walk, hsave (K, batch, save_tiles, D, N) indexed by the backward's walk-order tile number
  float *dsave, *hsave;
  int save_tiles;
  int D, N, R, Cp, kind, batch, ndir;
  long long Lseq;
  int I[4], O[4], rev[4];
  long long istride[4], ostride[4];   // y element strides of the inner / outer walk index
  int nsplit, tiles_per_split;
  int nst;     // TMA ring depth: as many LT-position stages as fit next to CTAS-1 other CTAs in shared memory
  int ablate;  // timing experiments, only in builds with -DSIGMA_SCAN_ABLATION (SIGMA_SCAN_ABLATE env):
               // 1 = no y store, 2 = no per-group prologue, 4 = no TMA reload
  int xc_dtype; // SIGMA_BF16 / SIGMA_F16: xc and y are bf16 / fp16; x_dbl, the state and the recurrence stay fp32.  With hsave
                // (the bf16 / fp16 training modes) the delta' slabs are bf16 / fp16 too and the recurrence runs on the rounded delta'
};

#ifdef SIGMA_SCAN_ABLATION
#define SIGMA_ABL(flags, m) (((flags) & (m)) != 0)
#else
#define SIGMA_ABL(flags, m) false
#endif

// xc_bytes: element size of the staged xc tile (4, or 2 for bf16 / fp16)
__host__ __device__ inline size_t ss2d_smem_bytes(int LT, int DT, int NST, int Cp, bool cross, int xc_bytes = 4) {
  const size_t stage = (size_t)LT * DT * xc_bytes + (size_t)LT * Cp * (cross ? 2 : 1) * sizeof(float);
  return NST * stage + 128 /*barriers + counters*/;
}

static __device__ float g_ss2d_sink[32];   // y of threads whose channel is >= D goes here (never read)

template <int N, int CPT, int RP>
struct Ss2dThread {
  float h[CPT][N], a2[CPT][N], W[CPT][RP];
  unsigned long long bias2[CPT];   // {dt bias, 0} as one 64-bit register pair: initial value of the dt_proj accumulator
  float Dv[CPT], sumdl[CPT];
  bool ok[CPT];
  int ablate;
};

// pair helpers on 64-bit register pairs (two scalar fp32 operations each, common.cuh)
__device__ __forceinline__ unsigned long long fma2_raw(unsigned long long a, unsigned long long b, unsigned long long c) {
  const f2 x = unpack2(a), y = unpack2(b), z = unpack2(c);
  return pack2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}

__device__ __forceinline__ unsigned long long mul2_raw(unsigned long long a, unsigned long long b) {
  const f2 x = unpack2(a), y = unpack2(b);
  return pack2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}

// delta' and u of the thread's channels for the G positions whose x_dbl rows start at `drow` (pointing at the
// dt_r part of the first row) and whose xc values start at `xrow` (this thread's first channel).  dt_r is read
// once per position (broadcast LDS.128) and used for all CPT channels; the dot product runs on fma2 pairs
// (one accumulator chain up to RP = 12, two beyond), softplus is branch-free (common.cuh).
// RND (the bf16 / fp16 training modes): delta' is rounded to XT (bf16 / fp16) here, before the recurrence uses it, so that the
// value the forward runs on is exactly the value it saves for the backward.
template <int N, int CPT, int RP, int G, bool RND = false, typename XT>
__device__ __forceinline__ void group_prologue(const Ss2dThread<N, CPT, RP> &t, const XT *xrow, const float *drow, int DT,
                                               float (&dl)[CPT][G], float (&u)[CPT][G]) {
  constexpr int Cp = 2 * N + RP;  // x_dbl row length: [B | C | dt_r padded to RP] (sigma_ss2d_padded_cp)
  constexpr bool TWO = RP >= 16;
  const int cstride = DT / CPT;
#pragma unroll
  for (int e = 0; e < G; ++e) {
    const float *row = drow + e * Cp;
    unsigned long long acc0[CPT], acc1[CPT];
#pragma unroll
    for (int c = 0; c < CPT; ++c) { acc0[c] = t.bias2[c]; acc1[c] = 0ull; }
#pragma unroll
    for (int q4 = 0; q4 < RP / 4; ++q4) {
      const float4 v = *reinterpret_cast<const float4 *>(row + 4 * q4);   // broadcast read, shared by CPT channels
#pragma unroll
      for (int c = 0; c < CPT; ++c) {
        acc0[c] = fma2_raw(pack2(t.W[c][4 * q4 + 0], t.W[c][4 * q4 + 1]), pack2(v.x, v.y), acc0[c]);
        if (TWO) {
          acc1[c] = q4 == 0 ? mul2_raw(pack2(t.W[c][2], t.W[c][3]), pack2(v.z, v.w))
                            : fma2_raw(pack2(t.W[c][4 * q4 + 2], t.W[c][4 * q4 + 3]), pack2(v.z, v.w), acc1[c]);
        } else {
          acc0[c] = fma2_raw(pack2(t.W[c][4 * q4 + 2], t.W[c][4 * q4 + 3]), pack2(v.z, v.w), acc0[c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
      const f2 s0 = unpack2(acc0[c]);
      float x = s0.x + s0.y;
      if (TWO) { const f2 s1 = unpack2(acc1[c]); x += s1.x + s1.y; }
      dl[c][e] = x;                                   // pre-activation; softplus below, two positions per softplus20x2
      u[c][e] = to_f32(xrow[e * DT + c * cstride]);
    }
  }
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
#pragma unroll
    for (int e = 0; e < G; e += 2) {
      const f2 sp = softplus20x2(dl[c][e], dl[c][e + 1]);
      dl[c][e] = RND ? to_f32(from_f32<XT>(sp.x)) : sp.x;
      dl[c][e + 1] = RND ? to_f32(from_f32<XT>(sp.y)) : sp.y;
    }
  }
}

// recurrence over `cnt` (<= G) positions of one group, in walk order (REV: descending tile rows).  `rb` = first
// x_dbl row of the group (B part), `rc` = same row in the tile C is read from, `yq` = y of the group's first WALKED
// position (this thread's channel), `ystep` = y elements from one walked position to the next (negative when REV):
// the address is a running pointer (one IMAD.WIDE per position) and the store is unconditional — a thread whose
// channel lies beyond D walks a one-element sink instead (kernel prologue), so there is no branch around the store.
// Per position B and C are read ONCE (2·N/4 broadcast LDS.128) and reused by the CPT channels of the thread;
// per channel and state pair: mul2 (exp arguments), 2 x MUFU.EX2, mul2 (delta·u·B), fma2 (h), fma2 (C·h).
template <int N, int CPT, int RP, int G, bool WITH_Y, bool REV, bool FULL, bool SAVE = false, typename XT = float, typename ST = float>
__device__ __forceinline__ void group_body(Ss2dThread<N, CPT, RP> &t, const float *rb, const float *rc, XT *yq,
                                           int ystep, int ycstride, const float (&dl)[CPT][G],
                                           const float (&u)[CPT][G], int cnt, ST *dq = nullptr) {
  constexpr int Cp = 2 * N + RP;
  constexpr int NCH = N >= 8 ? 2 : 1;   // independent C·h accumulator chains per channel
#pragma unroll
  for (int ii = 0; ii < G; ++ii) {
    const int i = REV ? G - 1 - ii : ii;
    if (FULL || i < cnt) {
      const float *pb = rb + i * Cp;
      const float *pc = rc + i * Cp;
      f2 yacc[CPT][NCH];
#pragma unroll
      for (int s4 = 0; s4 < N / 4; ++s4) {
        const float4 bv = *reinterpret_cast<const float4 *>(pb + 4 * s4);   // broadcast reads
        float4 cv = make_float4(0.f, 0.f, 0.f, 0.f);
        if (WITH_Y) cv = *reinterpret_cast<const float4 *>(pc + 4 * s4);
#pragma unroll
        for (int c = 0; c < CPT; ++c) {
          const float d = dl[c][i], du = dl[c][i] * u[c][i];
#pragma unroll
          for (int hp = 0; hp < 2; ++hp) {                                   // state pair (4·s4 + 2·hp, +1)
            const int s = 4 * s4 + 2 * hp;
            const f2 arg = mul2(f2{d, d}, f2{t.a2[c][s], t.a2[c][s + 1]});
            const f2 a = f2{ex2(arg.x), ex2(arg.y)};
            const f2 bb = mul2(f2{du, du}, hp == 0 ? f2{bv.x, bv.y} : f2{bv.z, bv.w});
            const f2 hn = fma2(a, f2{t.h[c][s], t.h[c][s + 1]}, bb);
            t.h[c][s] = hn.x; t.h[c][s + 1] = hn.y;
            if (WITH_Y) {
              const f2 cc = hp == 0 ? f2{cv.x, cv.y} : f2{cv.z, cv.w};
              const int ch = NCH == 2 ? hp : 0;
              const bool first = NCH == 2 ? s4 == 0 : (s4 == 0 && hp == 0);
              yacc[c][ch] = first ? mul2(hn, cc) : fma2(hn, cc, yacc[c][ch]);
            }
          }
        }
      }
#pragma unroll
      for (int c = 0; c < CPT; ++c) {
        if (WITH_Y) {
          float y = yacc[c][0].x + yacc[c][0].y;
          if (NCH == 2) y += yacc[c][1].x + yacc[c][1].y;
          if (SIGMA_ABL(t.ablate, 1)) t.sumdl[c] += y;
          else yq[c * ycstride] = from_f32<XT>(fmaf(t.Dv[c], u[c][i], y));
          if (SAVE) dq[c * ycstride] = from_f32<ST>(dl[c][i]);
        } else {
          t.sumdl[c] += dl[c][i];
        }
      }
    }
    if (WITH_Y) yq += ystep;
    if (SAVE) dq += ystep;
  }
}

// Everything a warp needs to walk its CTA's tiles; filled once in the kernel.
template <int N, int CPT, int RP, typename XT = float, typename ST = float>
struct Ss2dWalk {
  float *stages;
  uint64_t *full;
  uint32_t *done;
  XT *ybase;
  long long istride, ostride;
  int ystep;   // y elements from one walked position to the next (sign follows the walk direction; 0 on the sink)
  ST *dbase;           // SAVE: this thread's channel in the delta' slab of (k, b) (same addressing as ybase)
  float *hs_base;      // SAVE: hsave + (((k·batch + b)·save_tiles)·D + d)·N; tile tau16 adds tau16·D·N
  long long hs_stride; // D·N (0 on the sink)
  int TPO16, ntiles16; // 16-position blocks per inner walk line / in the whole walk (the backward's tile geometry)
  int stage_fl, xc_fl, dbl_fl, DT, nwarps, lane, ch;   // in floats (xc_fl: the xc tile's bytes / 4)
  int t0, t1, TPO, ntiles, I, nst;
  bool cross, rev;
};

// The tile loop of one warp.  The software pipeline over groups of G positions runs ACROSS tiles: while the
// recurrence of group g runs, delta'/u of group g+1 are computed — from the next tile's ring slot when g is the
// last group of its tile — so no prologue is exposed at a tile boundary and none is computed twice.
template <int N, int CPT, int RP, bool WITH_Y, bool REV, bool SAVE, bool RND, typename XT, typename ST, typename Request>
__device__ __forceinline__ void walk_tiles(Ss2dThread<N, CPT, RP> &t, const Ss2dWalk<N, CPT, RP, XT, ST> &w, Request &&request_tile) {
  constexpr int G = Ss2dCfg<N>::G, LT = Ss2dCfg<N>::LT;
  constexpr int Cp = 2 * N + RP;
  const int ycs = w.DT / CPT;

  // ring slot / phase and (outer index, inner tile) of the tile being opened advance incrementally: no division
  // or modulo per tile.  Tiles are walked in ascending tau; reversed directions map tau -> ntiles-1-tau.
  struct Tile { const XT *sXC; const float *sDB, *sDC; XT *ystart; ST *dstart; int npos, ng, tm16; };   // ystart: y of the tile's first WALKED group start
  int ost = 0, oph = 0;                                  // slot and phase parity of the next tile to open
  int tm0 = w.rev ? w.ntiles - 1 - w.t0 : w.t0;          // memory-order tile index of tile t0
  int oo = tm0 / w.TPO, oti = tm0 - oo * w.TPO;          // its (outer index, inner tile)
  auto open_tile = [&]() {   // waits for the next tile's TMA bytes; returns its pointers and advances the cursor
    if (!(SIGMA_ABL(t.ablate, 4) && oph)) mbar_spin(&w.full[ost], (uint32_t)oph);
    Tile T;
    T.sXC = reinterpret_cast<const XT *>(w.stages + ost * w.stage_fl);
    T.sDB = w.stages + ost * w.stage_fl + w.xc_fl;
    T.sDC = w.cross ? T.sDB + w.dbl_fl : T.sDB;
    const int i0 = oti * LT;
    T.npos = min(LT, w.I - i0);
    T.ng = (T.npos + G - 1) / G;
    const long long yoff = (long long)oo * w.ostride + (long long)(i0 + (REV ? T.ng * G - 1 : 0)) * w.istride;
    T.ystart = w.ybase + yoff;
    T.dstart = SAVE ? w.dbase + yoff : nullptr;
    T.tm16 = SAVE ? oo * w.TPO16 + (i0 >> 4) : 0;      // memory-order index of the tile's first 16-position block
    if (++ost == w.nst) { ost = 0; oph ^= 1; }
    if (w.rev) { if (--oti < 0) { oti = w.TPO - 1; --oo; } }
    else       { if (++oti == w.TPO) { oti = 0; ++oo; } }
    return T;
  };

  if (w.t0 >= w.t1) return;
  Tile cur = open_tile();
  int j = REV ? cur.ng - 1 : 0;   // walking backwards, a ragged group (npos % G) comes first
  float dl[CPT][G], u[CPT][G];
  group_prologue<N, CPT, RP, G, RND>(t, cur.sXC + j * G * w.DT + w.ch, cur.sDB + j * G * Cp + 2 * N, w.DT, dl, u);

  int rst = 0;                    // ring slot of the tile being processed
  const int gstep = G * w.ystep;  // y elements from one group's first walked position to the next group's
  XT *yp = cur.ystart;            // running y pointer: first walked position of the current group
  ST *dp = cur.dstart;
  for (int tau = w.t0; tau < w.t1; ++tau) {
    Tile nxt = cur;
    int jn = j;
#pragma unroll 1
    for (int g = 0; g < cur.ng; ++g) {
      // next group's delta'/u first, so its loads / dot products / softplus overlap this group's exponentials
      const XT *px;
      const float *pd;
      if (g + 1 < cur.ng) {
        jn = REV ? j - 1 : j + 1;
        px = cur.sXC + jn * G * w.DT + w.ch;
        pd = cur.sDB + jn * G * Cp + 2 * N;
      } else if (tau + 1 < w.t1) {
        nxt = open_tile();
        jn = REV ? nxt.ng - 1 : 0;
        px = nxt.sXC + jn * G * w.DT + w.ch;
        pd = nxt.sDB + jn * G * Cp + 2 * N;
      } else {                       // very last group of the walk: recompute the current one (result unused)
        px = cur.sXC + j * G * w.DT + w.ch;
        pd = cur.sDB + j * G * Cp + 2 * N;
      }
      float dln[CPT][G], un[CPT][G];
      const int cnt = cur.npos - j * G;
      const float *rb = cur.sDB + j * G * Cp;
      const float *rc = cur.sDC + j * G * Cp + N;
      // prologue(next) and body(current) are independent; keeping them in ONE basic block lets ptxas interleave
      // the prologue's FMA/LG2 work with the body's exponentials (it does not schedule across the cnt branch)
      if (SAVE) {
        // state entering a 16-position block of the walk (the backward's tile start): the block's first walked group
        const bool first = REV ? ((((j + 1) * G) & 15) == 0 || j == cur.ng - 1) : (((j * G) & 15) == 0);
        if (first && t.ok[0]) {
          const int tm16 = cur.tm16 + ((j * G) >> 4);
          float4 *hp = reinterpret_cast<float4 *>(w.hs_base + (long long)(REV ? w.ntiles16 - 1 - tm16 : tm16) * w.hs_stride);
#pragma unroll
          for (int q = 0; q < N / 4; ++q) hp[q] = make_float4(t.h[0][4 * q], t.h[0][4 * q + 1], t.h[0][4 * q + 2], t.h[0][4 * q + 3]);
        }
      }
      if (cnt >= G) {
        if (!SIGMA_ABL(t.ablate, 2)) group_prologue<N, CPT, RP, G, RND>(t, px, pd, w.DT, dln, un);
        else {
#pragma unroll
          for (int c = 0; c < CPT; ++c)
#pragma unroll
            for (int i = 0; i < G; ++i) { dln[c][i] = dl[c][i] * 1.0001f; un[c][i] = u[c][i]; }
        }
        group_body<N, CPT, RP, G, WITH_Y, REV, true, SAVE, XT, ST>(t, rb, rc, yp, w.ystep, ycs, dl, u, G, dp);
      } else {
        group_prologue<N, CPT, RP, G, RND>(t, px, pd, w.DT, dln, un);
        group_body<N, CPT, RP, G, WITH_Y, REV, false, SAVE, XT, ST>(t, rb, rc, yp, w.ystep, ycs, dl, u, cnt, dp);
      }
#pragma unroll
      for (int c = 0; c < CPT; ++c)
#pragma unroll
        for (int i = 0; i < G; ++i) { dl[c][i] = dln[c][i]; u[c][i] = un[c][i]; }
      j = jn;
      yp += gstep;
      if (SAVE) dp += gstep;
    }
    // this warp is done with the ring slot; the last of the CTA's warps to get here refills it
    __syncwarp();
    if (w.lane == 0 && tau + w.nst < w.t1) {
      const uint32_t old = smem_inc_acq_rel(&w.done[rst]);
      if ((old + 1) % (uint32_t)w.nwarps == 0) request_tile(tau + w.nst, rst);
    }
    if (++rst == w.nst) rst = 0;
    cur = nxt;
    yp = cur.ystart;
    dp = cur.dstart;
  }
}

// XT: element type of xc and y (float; __nv_bfloat16 in the bf16 inference and training modes, __half in the fp16 inference and
// training modes).
// TRAIN16 (the bf16 / fp16 training modes, XT = __nv_bfloat16 / __half): delta' is rounded to XT before the recurrence uses it —
// in the summary pass too, whose carries must describe the same recurrence — and the SAVE passes store that rounded delta'.
template <int N, int CPT, int RP, int MODE, bool SAVE, typename XT, bool TRAIN16>
__device__ __forceinline__ void ss2d_scan_body(const Ss2dParams &p) {
  static_assert(!SAVE || MODE != MODE_SUMMARY, "the summary pass has no final states to save");
  static_assert(!SAVE || sizeof(XT) == 4 || TRAIN16, "the fp32 training forward stores fp32");
  static_assert(!TRAIN16 || sizeof(XT) == 2, "the 16-bit training modes read and write 16-bit elements");
  using ST = std::conditional_t<TRAIN16, XT, float>;   // element type of the saved delta' slabs
  constexpr int LT = Ss2dCfg<N>::LT;
  constexpr bool WITH_Y = MODE != MODE_SUMMARY;
  const int NST = p.nst;

  extern __shared__ __align__(1024) unsigned char smem_raw[];  // TMA destinations need 128-byte alignment
  float *stages = reinterpret_cast<float *>(smem_raw);
  constexpr int Cp = 2 * N + RP;  // == p.Cp (checked on the host)
  const bool cross = p.kind == SIGMA_DIRS_CROSS;

  const int tid = threadIdx.x;
  const int NTC = blockDim.x;                // every warp computes; there is no producer warp
  const int DT = NTC * CPT;                  // channels per CTA: thread t owns channels t and t + NTC (CPT = 2)
  const int xc_fl = LT * DT * (int)sizeof(XT) / 4, dbl_fl = LT * Cp;
  const int stage_fl = xc_fl + dbl_fl * (cross ? 2 : 1);
  uint64_t *full = reinterpret_cast<uint64_t *>(stages + NST * stage_fl);
  uint32_t *done = reinterpret_cast<uint32_t *>(full + NST);   // per-slot count of warps done with the slot

  const int d0 = blockIdx.x * DT;
  const int k = cross ? 0 : blockIdx.y / p.nsplit;
  const int split = cross ? blockIdx.y : blockIdx.y - k * p.nsplit;
  const int b = blockIdx.z;
  const int half = p.batch >> 1;        // CROSS: images [0,half) are modality 0 (rgb), [half,batch) modality 1
  const int kw = cross ? (b >= half ? 1 : 0) : k;                 // which weight set (direction / modality)
  const int bC = cross ? (b >= half ? b - half : b + half) : b;   // C of the OTHER modality (vmamba.py:1530,1536)
  const int I = p.I[k], O = p.O[k];
  const bool rev = p.rev[k] != 0;
  const int TPO = (I + LT - 1) / LT, ntiles = O * TPO;
  const int t0 = split * p.tiles_per_split, t1 = min(ntiles, t0 + p.tiles_per_split);

  if (tid == 0) {
    for (int s = 0; s < NST; ++s) {
      mbar_init(&full[s], 1);           // one arrive (the requester's expect_tx) + the TMA bytes
      done[s] = 0;
    }
    fence_mbar_init();
  }
  __syncthreads();

  // One lane requests tile tau (its ring slot is known to be free): arm the slot's full barrier with the byte
  // count and issue the 2 (3) TMA loads.
  const uint32_t tx_bytes = (uint32_t)(stage_fl * sizeof(float));
  auto request_tile = [&](int tau, int st) {
    if (SIGMA_ABL(p.ablate, 4) && tau - t0 >= NST) return;
    float *dst = stages + st * stage_fl;
    const int tm = rev ? ntiles - 1 - tau : tau;
    const int o = tm / TPO, i0 = (tm - o * TPO) * LT;
    mbar_arrive_expect_tx(&full[st], tx_bytes);
    tma_load_4d(dst, &p.m_xc[k], &full[st], d0, i0, o, b);
    tma_load_4d(dst + xc_fl, &p.m_dbl[k], &full[st], 0, i0, o, b);
    if (cross) tma_load_4d(dst + xc_fl + dbl_fl, &p.m_dbl[k], &full[st], 0, i0, o, bC);
  };
  if (tid == 0) {
    tma_prefetch_desc(&p.m_xc[k]);
    tma_prefetch_desc(&p.m_dbl[k]);
    for (int tau = t0; tau < min(t1, t0 + NST); ++tau) request_tile(tau, tau - t0);
  }

  // ===== CPT channels per thread, all N states of each in registers =====
  Ss2dThread<N, CPT, RP> t;
  t.ablate = p.ablate;
  float *carry_row[CPT];
#pragma unroll
  for (int c = 0; c < CPT; ++c) {
    const int d = d0 + tid + c * NTC;
    t.ok[c] = d < p.D;
    const long long wd = (long long)kw * p.D + (t.ok[c] ? d : 0);
#pragma unroll
    for (int s = 0; s < N; ++s) {
      t.a2[c][s] = t.ok[c] ? p.A[wd * N + s] * kLog2e : 0.f;
      t.h[c][s] = 0.f;
    }
#pragma unroll
    for (int r = 0; r < RP; ++r) t.W[c][r] = (t.ok[c] && r < p.R) ? p.dtw[wd * p.R + r] : 0.f;
    {
      const float bias = t.ok[c] ? p.dtb[wd] : 0.f;
      asm volatile("mov.b64 %0, {%1, %2};" : "=l"(t.bias2[c]) : "f"(bias), "f"(0.f));   // opaque: stays a register pair
    }
    t.Dv[c] = t.ok[c] ? p.Ds[wd] : 0.f;
    t.sumdl[c] = 0.f;
    carry_row[c] = nullptr;
    if (MODE != MODE_SERIAL) {
      carry_row[c] = p.carry + ((((long long)b * p.ndir + k) * p.D + (t.ok[c] ? d : 0)) * p.nsplit + split) * 2 * N;
      if (MODE == MODE_APPLY && t.ok[c]) {
#pragma unroll
        for (int s = 0; s < N; ++s) t.h[c][s] = carry_row[c][N + s];
      }
    }
  }

  Ss2dWalk<N, CPT, RP, XT, ST> w;
  w.stages = stages; w.full = full; w.done = done;
  static_assert(CPT == 1, "the sink redirection below assumes one channel per thread");
  if (t.ok[0]) {
    w.ybase = reinterpret_cast<XT *>(p.y) + (((long long)k * p.batch + b) * p.Lseq) * p.D + d0 + tid;
    w.istride = p.istride[k]; w.ostride = p.ostride[k];
  } else {                       // channel beyond D (ragged last channel tile): every y address collapses onto the sink
    w.ybase = reinterpret_cast<XT *>(&g_ss2d_sink[tid & 31]);
    w.istride = 0; w.ostride = 0;
  }
  w.ystep = (int)(rev ? -w.istride : w.istride);
  w.dbase = nullptr; w.hs_base = nullptr; w.hs_stride = 0; w.TPO16 = 0; w.ntiles16 = 0;
  if (SAVE) {
    w.dbase = t.ok[0] ? reinterpret_cast<ST *>(p.dsave) + (w.ybase - reinterpret_cast<XT *>(p.y)) : reinterpret_cast<ST *>(w.ybase);          // same (K, batch, Lseq, D) addressing as y; sink otherwise
    w.TPO16 = (I + 15) >> 4;
    w.ntiles16 = O * w.TPO16;
    w.hs_stride = (long long)p.D * N;
    w.hs_base = p.hsave + ((((long long)k * p.batch + b) * p.save_tiles) * p.D + min(d0 + tid, p.D - 1)) * N;
  }
  w.stage_fl = stage_fl; w.xc_fl = xc_fl; w.dbl_fl = dbl_fl; w.DT = DT;
  w.nwarps = NTC >> 5; w.lane = tid & 31; w.ch = tid;
  w.t0 = t0; w.t1 = t1; w.TPO = TPO; w.ntiles = ntiles; w.I = I; w.nst = NST;
  w.cross = cross; w.rev = rev;

  if (rev) walk_tiles<N, CPT, RP, WITH_Y, true, SAVE, TRAIN16>(t, w, request_tile);
  else     walk_tiles<N, CPT, RP, WITH_Y, false, SAVE, TRAIN16>(t, w, request_tile);

  if (MODE == MODE_SUMMARY || SIGMA_ABL(p.ablate, 1)) {
#pragma unroll
    for (int c = 0; c < CPT; ++c) {
      if (t.ok[c] && carry_row[c] != nullptr) {
#pragma unroll
        for (int s = 0; s < N; ++s) {
          carry_row[c][s] = ex2(t.a2[c][s] * t.sumdl[c]);
          carry_row[c][N + s] = t.h[c][s];
        }
      }
    }
  }
}

template <int N, int CPT, int RP, int MODE, int CTAS, bool SAVE = false, typename XT = float>
__global__ void __launch_bounds__(32 * Ss2dCfg<N>::MAXW, CTAS) ss2d_scan_kernel(const __grid_constant__ Ss2dParams p) {
  static_assert(!SAVE || sizeof(XT) == 4, "the 16-bit training forwards are ss2d_scan_train16_kernel / ss2d_scan_train_fp16_kernel");
  ss2d_scan_body<N, CPT, RP, MODE, SAVE, XT, false>(p);
}

// the bf16 training mode: bf16 xc / y and a bf16 delta' that the recurrence itself runs on (see ss2d_scan_body)
template <int N, int CPT, int RP, int MODE, int CTAS, bool SAVE>
__global__ void __launch_bounds__(32 * Ss2dCfg<N>::MAXW, CTAS) ss2d_scan_train16_kernel(const __grid_constant__ Ss2dParams p) {
  ss2d_scan_body<N, CPT, RP, MODE, SAVE, __nv_bfloat16, true>(p);
}

// the fp16 training mode: the same with fp16 xc / y / delta' (a delta' below 2^-14 is stored subnormal and the recurrence runs on
// that value; past ±65504 a store gives ±inf)
template <int N, int CPT, int RP, int MODE, int CTAS, bool SAVE>
__global__ void __launch_bounds__(32 * Ss2dCfg<N>::MAXW, CTAS) ss2d_scan_train_fp16_kernel(const __grid_constant__ Ss2dParams p) {
  ss2d_scan_body<N, CPT, RP, MODE, SAVE, __half, true>(p);
}

// host-side launcher for one (N, CPT, RP) instantiation; defined per RP in ss2d_scan_rp*.cu.
// `nthreads` = threads per CTA (each owning CPT channels).
template <int N, int CPT, int RP>
int ss2d_launch(const Ss2dParams &p, int nthreads, int ctas, cudaStream_t stream);

}  // namespace sigma
