// stages.cuh -- the two data-parallel stages of one Gauss-Newton iteration of
// dvo::DenseTracker::match() as warp-level device functions over shared-memory tiles
// (used by the level kernel in tracker.cu).
//
//   stage A: computeResidualsSse + computeWeightsSse + computeScaleSse
//            (dense_tracking_impl.cpp:133-393, 657-707, 590-638)
//   stage B: computeCompleteDataLogLikelihood + Jacobians + normal equations
//            (dense_tracking_impl.cpp:406-425, dense_tracking.cpp:333-342, 448-476, least_squares.cpp:58-64)
//
// Data movement.  The reference image is cut into tiles of kTileW x kTileH pixels; a CTA owns whole
// strips (kTileH full image rows) and walks their tiles band by band.  For every tile a producer warp
// asks the bulk-copy engine (cp.async.bulk, the TMA unit) for
//   * the tile's REFERENCE TILE RECORD (common.cuh): its rows of (I, Zsel), its slice of the point-cloud
//     template and -- in stage B -- its rows of (Ix, Iy), contiguous in HBM: one copy, and
//   * the WINDOW of the current image the tile's bilinear taps fall into: its bounding box follows from
//     projecting the tile's four corner rays at the minimum and maximum depth of the tile (a projective map
//     keeps the convex hull), plus the one-pixel halo the central differences need: one copy per window row,
// into one of kStages shared-memory stage buffers and arms an mbarrier with the byte count; the seven
// consumer warps (warp q <-> tile row q) wait on it, compute from shared memory and release the buffer
// through a second mbarrier, on which the producer waits before it refills the buffer.  Nothing per pixel is
// written back: stage B recomputes the residual of stage A from the staged tile (same operations, same bits)
// instead of reading a record, so per pixel and iteration the kernel moves 8 (reference) + 8 x window overlap
// (current P0) bytes in stage A and 16 + 8 x overlap (current P2) in stage B.
// A tap outside the staged window (window larger than the buffer, point behind the camera, ...) is
// gathered from global memory by the same code through generic pointers: the window is a cache, never a
// correctness condition.
//
// Sums.  A warp owns an image row: the pairwise scale sums of the row leave it as one 12-float summary, the 28
// normal-equation values of the row through a fixed halving exchange (flush_row_partial).  Everything above a row is
// combined by the level kernel in an order fixed by the level's geometry (rows of a strip in order, strips in order,
// fp64), so results do not depend on how strips are spread over CTAs.
//
// The gradient channels of the current image are formed from the staged (I, Z) neighbours of each tap:
// (P[x+1] - P[x-1]) * 0.5 with clamped indices is exactly calculateDerivativeX/Y (rgbd_image.cpp:419-472);
// the factor 0.5 is a power of two and is folded into the constants that multiply the blended gradient,
// so every rounding step equals the one the precomputed gradient planes would give.
//
// All arithmetic that decides validity is explicit round-to-nearest fp32 in a fixed order (f32x2 pairs
// where two channels share an operation), mirrored bit for bit by the oracle's MIRROR mode; the per-thread
// accumulation along a row uses whatever contraction the compiler picks.
#pragma once
#include "common.cuh"
#include "f32x2.cuh"

namespace dvo_b200 {

constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kConsumerWarps = kTileH;                    // warp q walks row q of every tile
constexpr int kCtaThreads = (kConsumerWarps + 1) * 32;    // + one producer warp
#ifndef DVO_WIN_COLS
#define DVO_WIN_COLS 152
#endif
#ifndef DVO_WIN_ROWS
#define DVO_WIN_ROWS 24
#endif
#ifndef DVO_STAGES
#define DVO_STAGES 2
#endif
constexpr int kWinCols = DVO_WIN_COLS;                    // window capacity: kTileW + 24 columns
constexpr int kWinRows = DVO_WIN_ROWS;                    //                  kTileH + 17 rows
constexpr int kStages = DVO_STAGES;

// ---- mbarrier / bulk-copy primitives (PTX ISA 8.6, sm_90a) ------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.release.cta.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.release.cta.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
// try_wait may suspend the thread in hardware until the phase completes or a time limit passes; the explicit limit (ns)
// keeps the polling loop around it from spinning (0 = no hint, the default).
#ifndef DVO_TRYWAIT_HINT_NS
#define DVO_TRYWAIT_HINT_NS 0
#endif
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
#if DVO_TRYWAIT_HINT_NS > 0
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity), "r"((unsigned)DVO_TRYWAIT_HINT_NS)
      : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
#endif
  return ok != 0;
}
// Bounded wait: a lost transaction must never hang the GPU.  try_wait suspends in hardware for a
// system-dependent time before it reports failure, so the loop is not a busy spin.
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity, int* error_flag) {
  unsigned spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (((++spins) & 0xfffu) == 0u) {
      if (*reinterpret_cast<volatile int*>(error_flag)) break;
      if (spins > (1u << 24)) { atomicExch(error_flag, 2); break; }
    }
  }
}
// the same on 32-bit shared-window addresses (the consumers keep the pipe's base address in a register: going through
// generic pointers re-derives the shared window from special registers at every tile)
__device__ __forceinline__ bool mbar_try_wait_s(unsigned bar, unsigned parity) {
  unsigned ok;
#if DVO_TRYWAIT_HINT_NS > 0
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2, %3;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"((unsigned)DVO_TRYWAIT_HINT_NS)
      : "memory");
#else
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
#endif
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_s(unsigned bar, unsigned parity, int* error_flag) {
  unsigned spins = 0;
  while (!mbar_try_wait_s(bar, parity)) {
    if (((++spins) & 0xfffu) == 0u) {
      if (*reinterpret_cast<volatile int*>(error_flag)) break;
      if (spins > (1u << 24)) { atomicExch(error_flag, 2); break; }
    }
  }
}
__device__ __forceinline__ void mbar_arrive_s(unsigned bar) {
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.release.cta.shared::cta.b64 st, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ int4 lds_i4(unsigned addr) {
  int4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

// global -> shared bulk copy of `bytes` (multiple of 16, both addresses 16-byte aligned); completion is
// counted on `bar` (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cta.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// explicit 32-bit shared-memory loads (immediate offsets fold into the instruction; no generic-address arithmetic).
// volatile: they stay between the mbarrier wait that makes the tile visible and the arrive that releases it.
template <int kOff>
__device__ __forceinline__ f2 lds_f2(unsigned addr) {
  f2 v;
  asm volatile("ld.shared.b64 %0, [%1+%2];" : "=l"(v) : "r"(addr), "n"(kOff));
  return v;
}
__device__ __forceinline__ float lds_f32(unsigned addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ f2 lds_f2_at(unsigned addr) {
  f2 v;
  asm volatile("ld.shared.b64 %0, [%1];" : "=l"(v) : "r"(addr));
  return v;
}

// Loop-invariant addresses and constants that the compiler would otherwise re-derive from special registers and
// kernel parameters in every round (S2R + a dozen integer ops): pin them in a register.
__device__ __forceinline__ unsigned pin(unsigned v) { asm volatile("" : "+r"(v)); return v; }
__device__ __forceinline__ int pin(int v) { asm volatile("" : "+r"(v)); return v; }
__device__ __forceinline__ float pin(float v) { asm volatile("" : "+f"(v)); return v; }
template <typename T>
__device__ __forceinline__ const T* pin(const T* p) { asm volatile("" : "+l"(p)); return p; }

// ---- shared-memory stage buffers -----------------------------------------------------------------------
struct __align__(16) TileDesc {   // written by the producer before it arms the full barrier of the stage
  int skip;                // 1: no pixel of the tile can be valid (no reference depth, or the window misses the image)
  int origin;              // (row_lo * kWinCols + bx0) * 8: byte offset of image pixel (0, 0) relative to win[0][0], negated by the
                           // consumer; row_lo is the (virtual, -1 .. h) image row of window row 0, bx0 the column of window column 0
  int ulo, ucount;         // a tap (u0, v0) is served by the window iff (unsigned)(u0 - ulo) < ucount
  int vlo, vcount;         //                                       and (unsigned)(v0 - vlo) < vcount
  int exact;               // 1: the window holds the whole bounding box of the tile's taps -- no in-bounds tap can miss it
  int pad_;
};
struct __align__(128) StageBuf {
  // the reference tile record (common.cuh), filled by ONE bulk copy: stage A takes the first two members, stage B all three
  float2 ref0[kTileH][kTileW];       // (I, Zsel) rows of the tile
  float tx[kTileW];                  // point-cloud template of the tile's columns
  float2 ref1[kTileH][kTileW];       // (Ix, Iy) rows (stage B)
  float2 win[kWinRows][kWinCols];    // window of the current image (P0 in stage A, P2 in stage B)
};
static_assert(offsetof(StageBuf, tx) == kRecTx * sizeof(float2) && offsetof(StageBuf, ref1) == kRecP1 * sizeof(float2) &&
              offsetof(StageBuf, win) == kRecF2 * sizeof(float2), "StageBuf must mirror the reference tile record");
struct TilePipe {
  StageBuf buf[kStages];
  unsigned long long full[kStages], empty[kStages];
  TileDesc desc[kStages];
};
static_assert(sizeof(TileDesc) == 32 && offsetof(TilePipe, desc) % 16 == 0, "TileDesc is read as two 16-byte words");

// developer timing (build with -DDVO_PIPE_TIMING, run with DVO_B200_TIMING=1): cycles one warp of the CTA spends
// waiting on the pipeline.  Compiled out of the product build.
#ifdef DVO_PIPE_TIMING
struct PipeTiming {
  unsigned long long wait_full_a = 0, wait_full_b = 0, wait_empty = 0, produce = 0, rounds_a = 0, rounds_b = 0;
  unsigned long long tiles = 0, tiles_inexact = 0, tiles_skipped = 0, slow_rounds = 0, rounds = 0;
  bool on = false;
};
#define DVO_CLOCK(tm) ((tm).on ? clock64() : 0)
#define DVO_ADD(tm, field, v) do { if ((tm).on) (tm).field += (v); } while (0)
#else
struct PipeTiming {};
#define DVO_CLOCK(tm) 0ll
#define DVO_ADD(tm, field, v) do { } while (0)
#endif

// geometry of one pyramid level and this CTA's share of it
struct LevelGeom {
  int w, h, n, pitch;       // pixels, row pitch of the planes (float2)
  int nbands, nstrips;
  int strip0, strip_step, nmine;   // this CTA's strips: strip0 + k * strip_step, k = 0 .. nmine-1
};

// ---- per pair-iteration constants ---------------------------------------------------------------
struct StageConsts {
  f2 k0, k1, k2, k3;          // (kt[0],kt[4]) (kt[1],kt[5]) (kt[2],kt[6]) (kt[3],kt[7]): rows X and Y of K*T
  float k8, k9, k10, k11;     // row Z
  f2 Pa, Pb;                  // precision used for the weights: (P00,P01), (P10,P11)
  f2 cgh, cg, fxyh;           // (0.25 fx/255, 0.25 fy/255), (0.5 fx/255, 0.5 fy/255), (0.5 fx, 0.5 fy)  (dense_tracking.cpp:215-220)
  float c_i, ubx, uby;
  int first_iteration;
};

__device__ __forceinline__ void load_stage_consts(const PairState& st, const PairLevel& pl, int w, int h, bool weights_from_prev,
                                                  StageConsts& c) {
  // PairState is rewritten between stages by another SM (persistent kernel): read it through L2 (ld.cg)
  float kt[12], P[4];
#pragma unroll
  for (int i = 0; i < 12; ++i) kt[i] = __ldcg(&st.kt[i]);
  // stage A runs before P_k exists: `precision` still holds P_{k-1}; stage B runs after, P_{k-1} is in precision_prev
#pragma unroll
  for (int i = 0; i < 4; ++i) P[i] = weights_from_prev ? __ldcg(&st.precision_prev[i]) : __ldcg(&st.precision[i]);
  c.k0 = pk(kt[0], kt[4]); c.k1 = pk(kt[1], kt[5]); c.k2 = pk(kt[2], kt[6]); c.k3 = pk(kt[3], kt[7]);
  c.k8 = kt[8]; c.k9 = kt[9]; c.k10 = kt[10]; c.k11 = kt[11];
  c.Pa = pk(P[0], P[1]); c.Pb = pk(P[2], P[3]);
  const float cgx = __fdiv_rn(__fmul_rn(0.5f, pl.cfx), 255.0f), cgy = __fdiv_rn(__fmul_rn(0.5f, pl.cfy), 255.0f);
  c.cg = pk(cgx, cgy);
  c.cgh = pk(0.5f * cgx, 0.5f * cgy);                  // exact: the 0.5 of the central difference, folded in
  c.fxyh = pk(0.5f * pl.cfx, 0.5f * pl.cfy);
  c.c_i = 1.0f / 255.0f;
  c.ubx = pin((float)(w - 2)); c.uby = pin((float)(h - 2));
  c.first_iteration = __ldcg(&st.iteration) == 0;
}

// ---- producer duty: one warp stages the tiles of a stage ------------------------------------------------------
// Tiles are numbered per CTA since the kernel started (`t`): buffer = t % kStages, mbarrier phase parity =
// (t / kStages) & 1.  The warp waits until all consumers have released the buffer's previous tile.
//
// The window of a tile follows from eight projections (four corner rays x {zmin, zmax}): eight lanes.  The warp
// therefore prepares FOUR tiles at a time (lane >> 3 selects the tile), which also overlaps the global-memory
// latency of their depth ranges and template entries, and then issues the copies tile by tile; the two words
// that describe a window travel from the tile's lane group to the whole warp by shuffle.  (One tile per trip made
// the producer the slowest warp of the CTA in stage A: ~600 instructions and two dependent global loads per tile
// against ~500 instructions per consumer warp.)
template <bool kStageB>
__device__ __noinline__ void produce_tiles(TilePipe& tp, const PairLevel& pl, const LevelGeom& g, const StageConsts& c, unsigned tbase,
                                           int ntiles, int* error_flag, PipeTiming& tm) {
  const int lane = threadIdx.x & 31, sub = lane >> 3;
  const float2* cur = kStageB ? pl.c3 : pl.c0;
  int s_issue = g.strip0, b_issue = 0;       // tile i0 + k in issue order
  for (int i0 = 0; i0 < ntiles; i0 += 4) {
    const long long tp0 = DVO_CLOCK(tm);
    // ---- windows of tiles i0 .. i0+3: corner rays x {zmin, zmax} (lane & 7 selects the corner, lane >> 3 the tile) ----
    unsigned wordA, wordD;   // skip | exact << 1 | ncols << 2 | nrows << 10;  bx0 | (row_lo + 1) << 16
    {
      const int ii = min(i0 + sub, ntiles - 1);
      const int sd = ii / g.nbands;
      const int s = g.strip0 + sd * g.strip_step, b = ii - sd * g.nbands;
      const int y0 = s * kTileH, rows = min(kTileH, g.h - y0);
      const int x0 = b * kTileW, bw = min(kTileW, g.w - x0);
      const float2 zr = __ldg(pl.rrange + (size_t)s * g.nbands + b);
      const float txc = __ldg(pl.rtmpl + ((lane & 1) ? x0 + bw - 1 : x0));
      const float tyc = __ldg(pl.rtmpl + g.w + ((lane & 2) ? y0 + rows - 1 : y0));
      const bool has_depth = zr.x <= zr.y;          // false: no non-NaN reference depth, nothing is selected in this tile
      const float z = (lane & 4) ? zr.y : zr.x;
      const float px = txc * z, py = tyc * z;
      const f2 XY = fma2(c.k0, bc(px), fma2(c.k1, bc(py), fma2(c.k2, bc(z), c.k3)));
      const float Zt = fmaf(c.k8, px, fmaf(c.k9, py, fmaf(c.k10, z, c.k11)));
      const float iz = 1.0f / Zt;
      float umin = lo(XY) * iz, vmin = hi(XY) * iz, umax = umin, vmax = vmin;
      const bool front_lane = Zt > 1e-6f && umin == umin && vmin == vmin;
#pragma unroll
      for (int off = 1; off < 8; off <<= 1) {       // stays inside the aligned group of eight lanes
        umin = fminf(umin, __shfl_xor_sync(kFullMask, umin, off)); umax = fmaxf(umax, __shfl_xor_sync(kFullMask, umax, off));
        vmin = fminf(vmin, __shfl_xor_sync(kFullMask, vmin, off)); vmax = fmaxf(vmax, __shfl_xor_sync(kFullMask, vmax, off));
      }
      const bool front = ((__ballot_sync(kFullMask, front_lane) >> (sub * 8)) & 0xffu) == 0xffu;
      // clamp before the float -> int conversions; the slack below covers the rounding of the per-pixel projection
      umin = fmaxf(umin, -8.f); vmin = fmaxf(vmin, -8.f); umax = fminf(umax, (float)g.w + 8.f); vmax = fminf(vmax, (float)g.h + 8.f);
      int skip = 0, exact = 0, ncols = 0, nrows = 0, bx0 = 0, row_lo = 0;
      if (!has_depth) {
        skip = 1;
      } else if (!front) {
        // a corner behind the camera: the hull argument does not hold; stage no window, every tap is gathered
      } else if (umax < -1.f || vmax < -1.f || umin > (float)g.w || vmin > (float)g.h) {
        skip = 1;                       // the whole tile projects outside the current image
      } else {
        const int col_lo = max((int)floorf(umin) - 2, 0), col_hi = min((int)floorf(umax) + 3, g.w - 1);
        row_lo = max((int)floorf(vmin) - 2, -1);
        const int row_hi = min((int)floorf(vmax) + 3, g.h);
        bx0 = col_lo & ~1;
        ncols = (col_hi + 2 - bx0) & ~1;              // even count covering [bx0, col_hi]
        bool whole = true;
        if (ncols > kWinCols) { bx0 += ((ncols - kWinCols) / 2) & ~1; ncols = kWinCols; whole = false; }
        nrows = row_hi - row_lo + 1;
        if (nrows > kWinRows) { row_lo += (nrows - kWinRows) / 2; nrows = kWinRows; whole = false; }
        if (ncols < 4 || nrows < 4) { ncols = 0; nrows = 0; bx0 = 0; row_lo = 0; }
        else exact = whole ? 1 : 0;
      }
      wordA = (unsigned)skip | ((unsigned)exact << 1) | ((unsigned)ncols << 2) | ((unsigned)nrows << 10);
      wordD = (unsigned)bx0 | ((unsigned)(row_lo + 1) << 16);
    }
    DVO_ADD(tm, produce, DVO_CLOCK(tm) - tp0);
    // ---- issue: tile by tile, in order ----
    const int kmax = min(4, ntiles - i0);
    for (int k = 0; k < kmax; ++k) {
      const unsigned t = tbase + (unsigned)(i0 + k);
      const int bufi = t % kStages;
      StageBuf& sb = tp.buf[bufi];
      const unsigned wa = __shfl_sync(kFullMask, wordA, k * 8), wd = __shfl_sync(kFullMask, wordD, k * 8);
      const int s = s_issue, b = b_issue;
      if (++b_issue == g.nbands) { b_issue = 0; s_issue += g.strip_step; }
      const int skip = (int)(wa & 1u), ncols = (int)((wa >> 2) & 0xffu), nrows = (int)(wa >> 10);
      const int win_bx0 = (int)(wd & 0xffffu), win_row_lo = (int)(wd >> 16) - 1;
      TileDesc d;
      d.skip = skip; d.exact = (int)((wa >> 1) & 1u); d.pad_ = 0;
      d.origin = 0; d.ulo = 0; d.ucount = 0; d.vlo = 0; d.vcount = 0;
      if (ncols) {
        d.origin = (win_row_lo * kWinCols + win_bx0) * 8;
        // columns are clamped per tap (max(u0-1, 0), min(u0+2, w-1)); rows -1 and h are staged as replicas
        d.ulo = win_bx0 == 0 ? 0 : win_bx0 + 1;
        const int uhi = (win_bx0 + ncols - 1 >= g.w - 1) ? g.w - 2 : win_bx0 + ncols - 3;
        d.ucount = max(uhi - d.ulo + 1, 0);
        d.vlo = win_row_lo + 1;
        d.vcount = max(nrows - 3, 0);
      }
      const unsigned win_row_bytes = (unsigned)ncols * 8u;
      const unsigned rec_bytes = (unsigned)(kStageB ? kRecF2 : kRecP1) * 8u;       // stage A stops before the gradient rows
      const unsigned total = skip ? 0u : rec_bytes + (unsigned)nrows * win_row_bytes;
      // the descriptor is ready: now wait until the consumers have released the buffer's previous tile
      const long long tp1 = DVO_CLOCK(tm);
      mbar_wait(&tp.empty[bufi], ((t / kStages) & 1u) ^ 1u, error_flag);
      DVO_ADD(tm, wait_empty, DVO_CLOCK(tm) - tp1);
      DVO_ADD(tm, tiles, 1); DVO_ADD(tm, tiles_inexact, (!d.skip && !d.exact) ? 1 : 0); DVO_ADD(tm, tiles_skipped, d.skip ? 1 : 0);
      if (lane == 0) {
        tp.desc[bufi] = d;
        if (total) mbar_arrive_expect_tx(&tp.full[bufi], total);
        else mbar_arrive(&tp.full[bufi]);
      }
      __syncwarp();
      if (!skip) {
        if (lane < nrows) {
          const int yy = min(max(win_row_lo + lane, 0), g.h - 1);
          bulk_g2s(&sb.win[lane][0], cur + (size_t)yy * g.pitch + win_bx0, win_row_bytes, &tp.full[bufi]);
        }
        if (lane == 31) bulk_g2s(&sb.ref0[0][0], pl.r0 + (size_t)(s * g.nbands + b) * kRecF2, rec_bytes, &tp.full[bufi]);
      }
    }
  }
}

// ---- per-pixel geometry --------------------------------------------------------------------------------
// The residual record of one reference pixel (computeResidualsSse, dense_tracking_impl.cpp:133-393):
//   project_pixel : point (x,y,z) = (tx*z, ty*z, z); (X,Y,Z') = fma chains over the rows of K*T;
//                   (u,v) = (X,Y)*rcp_rn(Z'); bounds 0<=u<=w-2, 0<=v<=h-2; truncation -> tap index, weights.
//                   z = NaN (pixel not in the reference point list) fails the bounds test.
//   taps          : the four neighbours (stage B: twelve, for the central differences) from the staged window
//   blend         : bilinear blend, residual weights of dense_tracking.cpp:215-220, NaN test (line 261),
//                   occlusion test (line 275).  E = (e.i, e.z), G = (e.idx, e.idy), H = (e.zdx, e.zdy).
// Branch-free: a rejected point reads a safe location and is flagged invalid.
struct PixelProjection {
  f2 f, gq;        // (fu, fv), (gu, gv)
  float Zt;
  int u0, v0;      // upper-left tap
  bool inb;
};

__device__ __forceinline__ PixelProjection project_pixel(float tx, float ty, float z, const StageConsts& c) {
  PixelProjection p;
  const f2 pxy = mul2(pk(tx, ty), bc(z));
  const float px = lo(pxy), py = hi(pxy);
  const f2 XY = fma2(c.k0, bc(px), fma2(c.k1, bc(py), fma2(c.k2, bc(z), c.k3)));
  p.Zt = __fmaf_rn(c.k8, px, __fmaf_rn(c.k9, py, __fmaf_rn(c.k10, z, c.k11)));
  f2 uv = mul2(XY, bc(rcp_rn(p.Zt)));
  const float u = lo(uv), v = hi(uv);
  p.inb = u >= 0.f && u <= c.ubx && v >= 0.f && v <= c.uby;   // NaN compares false
  uv = p.inb ? uv : 0ull;
  // truncation without conversions: for 0 <= t < 2^23, RZ(t + 2^23) carries floor(t) in its mantissa
  const f2 t = add2_rz(uv, bc(8388608.0f));
  p.f = sub2(uv, sub2(t, bc(8388608.0f)));
  p.gq = sub2(bc(1.0f), p.f);
  p.u0 = __float_as_int(lo(t)) - 0x4b000000;
  p.v0 = __float_as_int(hi(t)) - 0x4b000000;
  return p;
}

#define DVO_BLEND2(fu, fv, gu, gv, c00, c10, c01, c11) \
  fma2(bc(fv), fma2(bc(fu), c11, mul2(bc(gu), c01)), mul2(bc(gv), fma2(bc(fu), c10, mul2(bc(gu), c00))))

__device__ __forceinline__ f2 ld_f2(const float2* p) { const float2 v = *p; return pk(v.x, v.y); }

// the staged window as one warp sees it during one tile
struct WinView {
  bool exact;                // no in-bounds tap of this tile can miss the window: skip the per-pixel test
  unsigned base;             // shared address of win[0][0] minus (row_lo * kWinCols + bx0) * 8: index with image coordinates
  unsigned safe;             // shared address of win[1][1]: where rejected points read
  const float2* plane;       // the same plane in global memory, for taps the window does not hold
  int ulo, ucount, vlo, vcount;
  int w, h, pitch;
};
constexpr int kWinRowBytes = kWinCols * 8;

struct Taps4 { f2 c00, c10, c01, c11; };
struct Taps12 { f2 c00, c10, c01, c11, l0, l1, r0, r1, t0, t1, b0, b1; };

// the rare path: some lane's taps lie outside the staged window -> generic loads, from the window or from global memory
// (inlined: a call inside the pixel loop would pin the accumulators to the calling convention's registers)
__device__ __forceinline__ void gather_taps4(const WinView& wv, int u0, int v0, bool inb, bool hit, Taps4& t) {
  const bool miss = inb && !hit;
  const unsigned sa = (inb && hit) ? wv.base + (unsigned)(v0 * kWinCols + u0) * 8u : wv.safe;
  const float2* p = miss ? wv.plane + (size_t)v0 * wv.pitch + u0 : reinterpret_cast<const float2*>(__cvta_shared_to_generic(sa));
  const int rp = miss ? wv.pitch : kWinCols;
  t.c00 = ld_f2(p); t.c10 = ld_f2(p + 1); t.c01 = ld_f2(p + rp); t.c11 = ld_f2(p + rp + 1);
}
__device__ __forceinline__ void gather_taps12(const WinView& wv, int u0, int v0, bool inb, bool hit, Taps12& t) {
  const bool miss = inb && !hit;
  const unsigned sa = (inb && hit) ? wv.base + (unsigned)(v0 * kWinCols + u0) * 8u : wv.safe;
  const float2* p = miss ? wv.plane + (size_t)v0 * wv.pitch + u0 : reinterpret_cast<const float2*>(__cvta_shared_to_generic(sa));
  const int rp = miss ? wv.pitch : kWinCols;
  const int up = (miss && v0 == 0) ? 0 : -rp;                     // the window holds rows -1 and h as replicas
  const int dn = (miss && v0 + 2 > wv.h - 1) ? rp : 2 * rp;
  const int dl = u0 > 0 ? 1 : 0, dr = u0 + 2 <= wv.w - 1 ? 2 : 1;
  t.c00 = ld_f2(p); t.c10 = ld_f2(p + 1); t.c01 = ld_f2(p + rp); t.c11 = ld_f2(p + rp + 1);
  t.t0 = ld_f2(p + up); t.t1 = ld_f2(p + up + 1); t.b0 = ld_f2(p + dn); t.b1 = ld_f2(p + dn + 1);
  t.l0 = ld_f2(p - dl); t.l1 = ld_f2(p + rp - dl); t.r0 = ld_f2(p + dr); t.r1 = ld_f2(p + rp + dr);
}

// depthStdDevZ (dense_tracking_impl.cpp:122-128)
__device__ __forceinline__ float depth_sigma(float z) {
  const float s = __fsub_rn(z, 0.4f);
  return __fmaf_rn(__fmul_rn(0.0019f, s), s, 0.0012f);
}

// Stage A pixel: (e.i, e.z) and validity from the four taps of (I, Z').
__device__ __forceinline__ bool residual_pixel(const PixelProjection& p, const WinView& wv, float Ir, float z, const StageConsts& c,
                                               float& ei, float& ez) {
  bool hit = true, any_miss = false;
  if (!wv.exact) {   // warp-uniform
    hit = (unsigned)(p.u0 - wv.ulo) < (unsigned)wv.ucount && (unsigned)(p.v0 - wv.vlo) < (unsigned)wv.vcount;
    any_miss = __any_sync(kFullMask, p.inb && !hit);
  }
  f2 c00, c10, c01, c11;
  if (!any_miss) {
    const unsigned a = p.inb ? wv.base + (unsigned)(p.v0 * kWinCols + p.u0) * 8u : wv.safe;
    c00 = lds_f2<0>(a); c10 = lds_f2<8>(a); c01 = lds_f2<kWinRowBytes>(a); c11 = lds_f2<kWinRowBytes + 8>(a);
  } else {
    Taps4 t;
    gather_taps4(wv, p.u0, p.v0, p.inb, hit, t);
    c00 = t.c00; c10 = t.c10; c01 = t.c01; c11 = t.c11;
  }
  const float fu = lo(p.f), fv = hi(p.f), gu = lo(p.gq), gv = hi(p.gq);
  const f2 IZ = DVO_BLEND2(fu, fv, gu, gv, c00, c10, c01, c11);
  const float Zc = hi(IZ);
  ez = __fsub_rn(Zc, p.Zt);
  ei = __fmaf_rn(c.c_i, lo(IZ), __fmul_rn(-c.c_i, Ir));
  return p.inb && Zc == Zc && ez > __fmul_rn(-20.0f, depth_sigma(z));
}

// Stage B pixel: the full record from twelve taps of (I, Z): centre 2x2, the columns left and right of it and the
// rows above and below it.
__device__ __forceinline__ bool record_pixel(const PixelProjection& p, const WinView& wv, float Ir, float z, f2 gref,
                                             const StageConsts& c, f2& E, f2& G, f2& H) {
  bool hit = true, any_miss = false;
  if (!wv.exact) {   // warp-uniform
    hit = (unsigned)(p.u0 - wv.ulo) < (unsigned)wv.ucount && (unsigned)(p.v0 - wv.vlo) < (unsigned)wv.vcount;
    any_miss = __any_sync(kFullMask, p.inb && !hit);
  }
  Taps12 t;
  if (!any_miss) {
    const unsigned a = p.inb ? wv.base + (unsigned)(p.v0 * kWinCols + p.u0) * 8u : wv.safe;
    t.c00 = lds_f2<0>(a); t.c10 = lds_f2<8>(a); t.c01 = lds_f2<kWinRowBytes>(a); t.c11 = lds_f2<kWinRowBytes + 8>(a);
    t.t0 = lds_f2<-kWinRowBytes>(a); t.t1 = lds_f2<-kWinRowBytes + 8>(a);
    t.b0 = lds_f2<2 * kWinRowBytes>(a); t.b1 = lds_f2<2 * kWinRowBytes + 8>(a);
    const unsigned al = a - (p.u0 > 0 ? 8u : 0u);                  // clamped column u0-1
    const unsigned ar = a + (p.u0 + 2 <= wv.w - 1 ? 16u : 8u);     // clamped column u0+2
    t.l0 = lds_f2<0>(al); t.l1 = lds_f2<kWinRowBytes>(al); t.r0 = lds_f2<0>(ar); t.r1 = lds_f2<kWinRowBytes>(ar);
  } else {
    gather_taps12(wv, p.u0, p.v0, p.inb, hit, t);
  }
  const float fu = lo(p.f), fv = hi(p.f), gu = lo(p.gq), gv = hi(p.gq);
  const f2 IZ = DVO_BLEND2(fu, fv, gu, gv, t.c00, t.c10, t.c01, t.c11);
  // 2 x central differences of (I, Z) at the four taps: x direction, y direction
  const f2 DX = DVO_BLEND2(fu, fv, gu, gv, sub2(t.c10, t.l0), sub2(t.r0, t.c00), sub2(t.c11, t.l1), sub2(t.r1, t.c01));
  const f2 DY = DVO_BLEND2(fu, fv, gu, gv, sub2(t.c01, t.t0), sub2(t.c11, t.t1), sub2(t.b0, t.c00), sub2(t.b1, t.c10));
  const float Zc = hi(IZ);
  const float ez = __fsub_rn(Zc, p.Zt);
  const float ei = __fmaf_rn(c.c_i, lo(IZ), __fmul_rn(-c.c_i, Ir));
  E = pk(ei, ez);
  G = fma2(c.cgh, pk(lo(DX), lo(DY)), mul2(c.cg, gref));
  H = mul2(c.fxyh, pk(hi(DX), hi(DY)));
  // dense_tracking_impl.cpp:261: any NaN among the eight blended lanes rejects the point
  const f2 nn = add2(add2(IZ, DX), DY);
  const float probe = lo(nn) + hi(nn);
  return p.inb && probe == probe && ez > __fmul_rn(-20.0f, depth_sigma(z));
}

// ---- pairwise scale sum ---------------------------------------------------------------------------
// computeScaleSse (dense_tracking_impl.cpp:590-638) walks the compacted residual list two at a time
// and, because lines 614-615 re-use the low half of the register, adds (w_{2j} + w_{2j+1}) r_{2j} r_{2j}^T
// for every pair plus w_n r_n r_n^T for an odd tail.  That needs, per valid point, the parity of its
// rank in row-major order and the weight of the next valid point.  A contiguous run of pixels is
// summarised by a segment record: the sums under both hypotheses for the parity of its first point
// (S0: the first valid point is a pair leader, S1: it is a follower), its first valid weight and its
// last valid point (a leader whose partner lies in the next run).  Runs combine associatively.
template <typename T>
struct SegT {
  long long n;
  T S0[3], S1[3];
  T wf, wl, ol[3];
};

template <typename T, typename A, typename B>
__host__ __device__ __forceinline__ SegT<T> combine_seg(const A& a, const B& b) {
  SegT<T> r;
  r.n = (long long)a.n + (long long)b.n;
  int hb0 = (int)(a.n & 1), hb1 = (int)((a.n + 1) & 1);
  bool link0 = a.n > 0 && b.n > 0 && (((a.n - 1) & 1) == 0);   // hypothesis 0: last point of a is a leader
  bool link1 = a.n > 0 && b.n > 0 && ((a.n & 1) == 0);         // hypothesis 1
  for (int k = 0; k < 3; ++k) {
    T bs0 = hb0 ? (T)b.S1[k] : (T)b.S0[k];
    T bs1 = hb1 ? (T)b.S1[k] : (T)b.S0[k];
    r.S0[k] = (T)a.S0[k] + bs0 + (link0 ? ((T)a.wl + (T)b.wf) * (T)a.ol[k] : (T)0);
    r.S1[k] = (T)a.S1[k] + bs1 + (link1 ? ((T)a.wl + (T)b.wf) * (T)a.ol[k] : (T)0);
  }
  r.wf = a.n > 0 ? (T)a.wf : (T)b.wf;
  if (b.n > 0) { r.wl = (T)b.wl; for (int k = 0; k < 3; ++k) r.ol[k] = (T)b.ol[k]; }
  else         { r.wl = (T)a.wl; for (int k = 0; k < 3; ++k) r.ol[k] = (T)a.ol[k]; }
  return r;
}

constexpr int kSegExportFloats = 12;   // n (as int bits), S0[3], S1[3], wf, wl, ol[3]

__device__ __forceinline__ SegT<double> load_seg_export(const float* e) {
  SegT<double> s;
  // written by other warps / SMs in the same kernel: read through L2
  float v[kSegExportFloats];
#pragma unroll
  for (int i = 0; i < kSegExportFloats; ++i) v[i] = __ldcg(e + i);
  s.n = __float_as_int(v[0]);
  s.S0[0] = v[1]; s.S0[1] = v[2]; s.S0[2] = v[3];
  s.S1[0] = v[4]; s.S1[1] = v[5]; s.S1[2] = v[6];
  s.wf = v[7]; s.wl = v[8]; s.ol[0] = v[9]; s.ol[1] = v[10]; s.ol[2] = v[11];
  return s;
}

// Strip summaries.  Everything above a row is combined in an order that depends only on the level's geometry, never on how
// the strips are spread over CTAs: the rows of a strip in order (one thread), the strips of the level by
// combine_strip_exports_warp (fixed chunks per lane, then an in-order tree), all in fp64 without intermediate rounding.
// Results are therefore bit-identical whatever the squad size: a batch of any size returns what single alignments return.
constexpr int kStripExportDoubles = 12;   // n, S0[3], S1[3], wf, wl, ol[3]
__device__ __forceinline__ void store_strip_export(const SegT<double>& s, double* e) {
  e[0] = (double)s.n;
  for (int k = 0; k < 3; ++k) { e[1 + k] = s.S0[k]; e[4 + k] = s.S1[k]; e[9 + k] = s.ol[k]; }
  e[7] = s.wf; e[8] = s.wl;
}
__device__ __forceinline__ SegT<double> load_strip_export(const double* e) {
  SegT<double> s;
  double v[kStripExportDoubles];
#pragma unroll
  for (int i = 0; i < kStripExportDoubles; ++i) v[i] = __ldcg(e + i);     // written by other SMs in the same kernel
  s.n = (long long)v[0];
  s.S0[0] = v[1]; s.S0[1] = v[2]; s.S0[2] = v[3];
  s.S1[0] = v[4]; s.S1[1] = v[5]; s.S1[2] = v[6];
  s.wf = v[7]; s.wl = v[8]; s.ol[0] = v[9]; s.ol[1] = v[10]; s.ol[2] = v[11];
  return s;
}
// one thread: rows [y0, y1) of one strip, in order -> the strip's summary; row_base[y] = valid points of the strip before row y
__device__ __forceinline__ void combine_strip_rows(const float* row_exports, int y0, int y1, int* row_base, double* strip_export) {
  SegT<double> acc;
  acc.n = 0; acc.wf = acc.wl = 0;
  for (int k = 0; k < 3; ++k) acc.S0[k] = acc.S1[k] = acc.ol[k] = 0;
#pragma unroll
  for (int k = 0; k < kTileH; ++k) {     // fixed trip count: the rows' loads are independent and overlap
    const int y = y0 + k;
    if (y < y1) {
      const SegT<double> r = load_seg_export(row_exports + (size_t)y * kSegExportFloats);
      row_base[y] = (int)acc.n;
      acc = combine_seg<double>(acc, r);
    }
  }
  store_strip_export(acc, strip_export);
}

// scratch of one warp-wide in-order combine
struct SegCombineSmem {
  SegT<double> lanes[32];
  long long lane_base[32];
};

// One warp combines the `count` strip summaries of a level, in order, into one; base_out[0 .. count] = exclusive prefix of the
// strips' valid counts
// (base_out[count] = all valid points).
__device__ __forceinline__ SegT<double> combine_strip_exports_warp(const double* e, int count, int* base_out, SegCombineSmem& sm) {
  const int lane = threadIdx.x & 31;
  const int chunk = (count + 31) / 32;
  const int t0 = min(lane * chunk, count), t1 = min(t0 + chunk, count);
  SegT<double> acc;
  acc.n = 0; acc.wf = acc.wl = 0;
  for (int k = 0; k < 3; ++k) acc.S0[k] = acc.S1[k] = acc.ol[k] = 0;
  for (int t = t0; t < t1; ++t) acc = combine_seg<double>(acc, load_strip_export(e + (size_t)t * kStripExportDoubles));
  sm.lanes[lane] = acc;
  {   // exclusive prefix of the lane counts
    long long incl = acc.n;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      long long v = __shfl_up_sync(kFullMask, incl, off);
      if (lane >= off) incl += v;
    }
    sm.lane_base[lane] = incl - acc.n;
  }
  __syncwarp();
  for (int off = 1; off < 32; off <<= 1) {   // in-order tree combine
    if ((lane & (2 * off - 1)) == 0) sm.lanes[lane] = combine_seg<double>(sm.lanes[lane], sm.lanes[lane + off]);
    __syncwarp();
  }
  long long run = sm.lane_base[lane];
  for (int t = t0; t < t1; ++t) {
    base_out[t] = (int)run;
    run += (long long)__ldcg(e + (size_t)t * kStripExportDoubles);
  }
  const SegT<double> all = sm.lanes[0];
  if (lane == 31) base_out[count] = (int)all.n;
  __syncwarp();
  return all;
}

// Student-t weight of computeWeightsSse (dense_tracking_impl.cpp:657-707): w = 7 / (5 + r^T P r), nu = 5;
// w = 1 on the first iteration of a level (dense_tracking.cpp:286-289).
__device__ __forceinline__ float student_weight(const StageConsts& c, float ei, float ez) {
  if (c.first_iteration) return 1.0f;
  const f2 q = fma2(bc(ez), c.Pb, mul2(bc(ei), c.Pa));        // (ei P00 + ez P10, ei P01 + ez P11)
  const float d = fmaf(lo(q), ei, hi(q) * ez);
  return 7.0f * rcp_fast(5.0f + d);
}

// Running state of the pairwise scale sum of one image row walked by one warp (see the comment above SegT).
// The row's sums are accumulated per lane in fp32 ((all, alternating-sign) packed per component) and leave the
// warp once per row; everything after that (rows -> CTA -> squad) is combined in fp64, so the result does not
// depend on how the rows are spread over CTAs.
struct ScaleState {
  f2 acc0, acc1, acc2;       // (sum, sum with the sign of the rank parity) of s * r r^T components 00, 01, 11
  float pw, po0, po1, po2;   // pending leader: the last valid point seen, waiting for the next valid weight
  float wfirst;
  int psign, cnt;
  bool pend;
};

__device__ __forceinline__ void scale_state_init(ScaleState& s) {
  s.acc0 = s.acc1 = s.acc2 = 0ull;
  s.pw = s.po0 = s.po1 = s.po2 = 0.f; s.wfirst = 0.f; s.psign = 0; s.cnt = 0; s.pend = false;
}

// Adds the 32 points {pixel base+lane: (v, w, ei, ez)} to the state.
__device__ __forceinline__ void scale_round32(ScaleState& st, int lane, unsigned lt_mask, bool v, float w, float ei, float ez) {
  const unsigned m = __ballot_sync(kFullMask, v);
  if (m == 0u) return;
  float w_first, wn, xi, xz;
  bool next;
  int sg;
  if (m == kFullMask) {   // the common round: every point valid, the next valid point is the next lane
    w_first = __shfl_sync(kFullMask, w, 0);
    wn = __shfl_down_sync(kFullMask, w, 1);
    next = lane != 31;
    sg = (int)((unsigned)(st.cnt + lane) << 31);
    xi = ei; xz = ez;
  } else {
    w_first = __shfl_sync(kFullMask, w, __ffs(m) - 1);              // first valid weight of the round
    const unsigned above = (m >> lane) >> 1;
    wn = __shfl_sync(kFullMask, w, above ? lane + __ffs(above) : lane);
    next = above != 0u;
    sg = (int)((unsigned)(st.cnt + __popc(m & lt_mask)) << 31);     // sign bit set for odd rank
    // rejected points carry garbage (possibly NaN) residuals: zero them so that 0 * outer stays 0
    xi = v ? ei : 0.f; xz = v ? ez : 0.f;
  }
  if (st.cnt == 0) st.wfirst = w_first;
  {   // the pending leader of an earlier round pairs with the first valid point of this round
    const float s = st.pend ? st.pw + w_first : 0.f;
    const f2 ss = pk(s, __int_as_float(__float_as_int(s) ^ st.psign));
    st.acc0 = fma2(ss, bc(st.po0), st.acc0); st.acc1 = fma2(ss, bc(st.po1), st.acc1); st.acc2 = fma2(ss, bc(st.po2), st.acc2);
  }
  const float a0 = xi * xi, a1 = xi * xz, a2 = xz * xz;
  const float s = (v && next) ? w + wn : 0.f;
  const f2 ss = pk(s, __int_as_float(__float_as_int(s) ^ sg));
  st.acc0 = fma2(ss, bc(a0), st.acc0); st.acc1 = fma2(ss, bc(a1), st.acc1); st.acc2 = fma2(ss, bc(a2), st.acc2);
  // new pending leader: the last valid point of the round (the values only matter in the lane that has `pend`)
  st.pend = v && !next;
  st.pw = w; st.po0 = a0; st.po1 = a1; st.po2 = a2; st.psign = sg;
  st.cnt += __popc(m);
}

// warp-reduce the sums and write the segment summary (kSegExportFloats floats)
__device__ __forceinline__ void scale_state_export(ScaleState& st, int lane, float* seg_out) {
  float all0 = lo(st.acc0), alt0 = hi(st.acc0), all1 = lo(st.acc1), alt1 = hi(st.acc1), all2 = lo(st.acc2), alt2 = hi(st.acc2);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    all0 += __shfl_xor_sync(kFullMask, all0, off); alt0 += __shfl_xor_sync(kFullMask, alt0, off);
    all1 += __shfl_xor_sync(kFullMask, all1, off); alt1 += __shfl_xor_sync(kFullMask, alt1, off);
    all2 += __shfl_xor_sync(kFullMask, all2, off); alt2 += __shfl_xor_sync(kFullMask, alt2, off);
  }
  // leaders at even local rank belong to hypothesis 0, odd to hypothesis 1: S0 = (all + alt)/2, S1 = (all - alt)/2
  if (lane == 0) {
    seg_out[0] = __int_as_float(st.cnt);
    seg_out[1] = (float)(0.5 * ((double)all0 + (double)alt0)); seg_out[2] = (float)(0.5 * ((double)all1 + (double)alt1));
    seg_out[3] = (float)(0.5 * ((double)all2 + (double)alt2));
    seg_out[4] = (float)(0.5 * ((double)all0 - (double)alt0)); seg_out[5] = (float)(0.5 * ((double)all1 - (double)alt1));
    seg_out[6] = (float)(0.5 * ((double)all2 - (double)alt2));
    seg_out[7] = st.wfirst;
    if (st.cnt == 0) { seg_out[8] = 0.f; seg_out[9] = 0.f; seg_out[10] = 0.f; seg_out[11] = 0.f; }
  }
  if (st.pend) {   // exactly one lane when cnt > 0: the last valid point of the segment
    seg_out[8] = st.pw; seg_out[9] = st.po0; seg_out[10] = st.po1; seg_out[11] = st.po2;
  }
}

// ---- consumers ------------------------------------------------------------------------------------------------
// `bufs`: shared-window address of the stage buffer; TileDesc as the two 16-byte words it is stored as
__device__ __forceinline__ WinView make_view(unsigned bufs, const int4& d0, const int4& d1, const float2* plane, int w, int h, int pitch) {
  WinView wv;
  const unsigned w0 = bufs + (unsigned)offsetof(StageBuf, win);
  wv.base = pin(w0 - (unsigned)d0.y);                       // TileDesc: {skip, origin, ulo, ucount}, {vlo, vcount, exact, pad}
  wv.safe = pin(w0 + (unsigned)((kWinCols + 1) * 8));
  wv.plane = plane;
  wv.exact = d1.z != 0;
  wv.ulo = d0.z; wv.ucount = d0.w; wv.vlo = d1.x; wv.vcount = d1.y;
  wv.w = w; wv.h = h; wv.pitch = pitch;
  return wv;
}
// Stage A over this CTA's strips: warp q walks image row strip*kTileH + q band by band, carries the pairwise
// scale state across the bands (they are consecutive pixels of the row) and writes one segment summary per row
// to row_exports[y * kSegExportFloats].  Warp kConsumerWarps is the producer: it stages the same tiles, kStages ahead.
__device__ __forceinline__ void stage_a_run(TilePipe& tp, const PairLevel& pl, const LevelGeom& g, const StageConsts& c,
                                            float* row_exports, unsigned& tile_count, int* error_flag, PipeTiming& tm) {
  const int lane = threadIdx.x & 31, q = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int ntiles = g.nmine * g.nbands;
  const unsigned tbase = tile_count;
  tile_count += ntiles;
  if (q == kConsumerWarps) {   // the producer warp
    produce_tiles<false>(tp, pl, g, c, tbase, ntiles, error_flag, tm);
    return;
  }
  int i = 0;
  // loop invariants in registers (the level geometry otherwise comes from constant memory through a dynamic index)
  const unsigned tp_s = pin(smem_u32(&tp));
  const unsigned my_ref = pin((unsigned)(offsetof(StageBuf, ref0) + (q * kTileW + lane) * 8));
  const unsigned my_tx = pin((unsigned)(offsetof(StageBuf, tx) + lane * 4));
  const int gw = pin(g.w), gh = pin(g.h), gnb = pin(g.nbands), gpitch = g.pitch;
  for (int sk = 0, s = g.strip0; sk < g.nmine; ++sk, s += g.strip_step) {
    const int y = s * kTileH + q;
    const bool row_ok = y < gh;
    const float ty = __ldg(pl.rtmpl + gw + min(y, gh - 1));
    ScaleState ss;
    scale_state_init(ss);
    for (int b = 0; b < gnb; ++b, ++i) {
      const unsigned t = tbase + i;
      const unsigned bufi = t % kStages;
      const int x0 = b * kTileW, bw = min(kTileW, gw - x0);
      const long long tw0 = DVO_CLOCK(tm);
      mbar_wait_s(tp_s + (unsigned)offsetof(TilePipe, full) + bufi * 8u, (t / kStages) & 1u, error_flag);
      DVO_ADD(tm, wait_full_a, DVO_CLOCK(tm) - tw0);
      const unsigned bufs = tp_s + bufi * (unsigned)sizeof(StageBuf);
      const int4 d0 = lds_i4(tp_s + (unsigned)offsetof(TilePipe, desc) + bufi * 32u);
      if (row_ok && !d0.x) {
        const int4 d1 = lds_i4(tp_s + (unsigned)offsetof(TilePipe, desc) + bufi * 32u + 16u);
        const WinView wv = make_view(bufs, d0, d1, pl.c0, gw, gh, gpitch);
        const int nr = (bw + 31) >> 5;
        unsigned refa = bufs + my_ref;
        unsigned txa = bufs + my_tx;
        const int xlim = bw - lane;        // lane's column r*32+lane is inside the band iff r*32 < xlim
        // two rounds per trip: their projection / tap / blend chains are independent and interleave
#pragma unroll 1
        for (int r = 0; r < nr; r += 2, refa += 512, txa += 256) {
          const bool second = r + 1 < nr;                       // warp-uniform
          const f2 rz0 = lds_f2_at(refa);
          const f2 rz1 = second ? lds_f2_at(refa + 256) : pk(0.f, __int_as_float(0x7fc00000));
          const float tx0 = lds_f32(txa), tx1 = second ? lds_f32(txa + 128) : 0.f;
          float z0 = hi(rz0), z1 = hi(rz1);
          if (bw < kTileW) {   // past a partial band: not this band's pixels
            z0 = (r * 32 < xlim) ? z0 : __int_as_float(0x7fc00000);
            z1 = (r * 32 + 32 < xlim) ? z1 : __int_as_float(0x7fc00000);
          }
          const PixelProjection p0 = project_pixel(tx0, ty, z0, c);
          const PixelProjection p1 = project_pixel(tx1, ty, z1, c);
          float ei0, ez0, ei1, ez1;
          const bool v0 = residual_pixel(p0, wv, lo(rz0), z0, c, ei0, ez0);
          const bool v1 = residual_pixel(p1, wv, lo(rz1), z1, c, ei1, ez1);
          const float w0 = student_weight(c, ei0, ez0), w1 = student_weight(c, ei1, ez1);
          scale_round32(ss, lane, lt_mask, v0, w0, ei0, ez0);
          scale_round32(ss, lane, lt_mask, v1, w1, ei1, ez1);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive_s(tp_s + (unsigned)offsetof(TilePipe, empty) + bufi * 8u);
    }
    if (row_ok) scale_state_export(ss, lane, row_exports + (size_t)y * kSegExportFloats);
  }
}

// ---- stage B -----------------------------------------------------------------------------------------
struct StageBConsts {
  float P00, P01, P10, P11;   // P_k
  float l, wd0, wd1;          // P_k = [1 l; 0 1]^T-style factors, see stage_b_pixel
};

constexpr int kNormalValues = 28;   // log-likelihood sum, 21 upper-triangular A (row-major), 6 b

// Accumulators of stage B for one thread.  A is kept as pairs of adjacent columns of one row
// (A[r][2c], A[r][2c+1]); rows 1, 3 and 5 carry one redundant lower-triangle entry so that every
// update is one fma2 of a broadcast row factor with a column pair.
struct StageBAcc;
__device__ __forceinline__ void stage_b_values(const StageBAcc& acc, float out[]);
struct StageBAcc {
  f2 r0[3], r1[3], r2[2], r3[2], r4, r5;   // 12 pairs
  f2 b[3];
  float llsum;     // sum of log2(1 + 0.2 r^T P r) over this thread's kept points
};

__device__ __forceinline__ void stage_b_init(StageBAcc& a) {
#pragma unroll
  for (int i = 0; i < 3; ++i) { a.r0[i] = 0; a.r1[i] = 0; a.b[i] = 0; }
  a.r2[0] = a.r2[1] = a.r3[0] = a.r3[1] = a.r4 = a.r5 = 0;
  a.llsum = 0.f;
}

// A += u v^T (upper triangle, column pairs) and b += u * s for one 6-vector given as three pairs V,
// with u = V * wd.
__device__ __forceinline__ void stage_b_rank1(StageBAcc& acc, const f2 V[3], float wd, float s) {
  const f2 U0 = mul2(V[0], bc(wd)), U1 = mul2(V[1], bc(wd)), U2 = mul2(V[2], bc(wd));
  const float u0 = lo(U0), u1 = hi(U0), u2 = lo(U1), u3 = hi(U1), u4 = lo(U2), u5 = hi(U2);
  acc.r0[0] = fma2(bc(u0), V[0], acc.r0[0]); acc.r0[1] = fma2(bc(u0), V[1], acc.r0[1]); acc.r0[2] = fma2(bc(u0), V[2], acc.r0[2]);
  acc.r1[0] = fma2(bc(u1), V[0], acc.r1[0]); acc.r1[1] = fma2(bc(u1), V[1], acc.r1[1]); acc.r1[2] = fma2(bc(u1), V[2], acc.r1[2]);
  acc.r2[0] = fma2(bc(u2), V[1], acc.r2[0]); acc.r2[1] = fma2(bc(u2), V[2], acc.r2[1]);
  acc.r3[0] = fma2(bc(u3), V[1], acc.r3[0]); acc.r3[1] = fma2(bc(u3), V[2], acc.r3[1]);
  acc.r4 = fma2(bc(u4), V[2], acc.r4);
  acc.r5 = fma2(bc(u5), V[2], acc.r5);
  acc.b[0] = fma2(U0, bc(s), acc.b[0]); acc.b[1] = fma2(U1, bc(s), acc.b[1]); acc.b[2] = fma2(U2, bc(s), acc.b[2]);
}

// One valid point: log-likelihood term and normal equations with W = w * P_k.
// With l = P01/P00, d0 = P00, d1 = P11 - P01^2/P00:
//   J^T P J = d0 j0' j0'^T + d1 J1 J1^T,  j0' = J0 + l J1,     J^T P r = d0 j0' (r0 + l r1) + d1 J1 r1
// so each point contributes two rank-1 updates.  J rows at the untransformed reference point
// (dense_tracking.cpp:448-476): J0 = gx a + gy b, J1 = hx a + hy b - c with
//   a = [1/z, 0, -x/z^2, a2 y, 1 - a2 x, -y/z], b = [0, 1/z, -y/z^2, b2 y - 1, -a3, x/z], c = [0, 0, 1, y, -x, 0].
// Branch-free: a rejected point arrives with wgt = 0 and finite stand-in inputs, so it adds exact zeros.
__device__ __forceinline__ void stage_b_pixel(StageBAcc& acc, const StageBConsts& c, float wgt, bool keep, float ei, float ez, f2 G,
                                              f2 H, float z, float tx, float ty) {
  // log-likelihood term: log(1 + 0.2 r^T P r); one MUFU.LG2 per point, scaled by ln 2 once at the end
  const float d = (ei * c.P00 + ez * c.P10) * ei + (ei * c.P01 + ez * c.P11) * ez;
  acc.llsum += __log2f(keep ? fmaf(0.2f, d, 1.0f) : 1.0f);
  const float px = tx * z, py = ty * z;
  const float zi = rcp_fast(z), zs = zi * zi;
  const float a2 = -px * zs, b2 = -py * zs;
  const float a3 = a2 * py;
  const f2 A23 = pk(a2, a3), B23 = pk(b2, fmaf(b2, py, -1.0f));
  const f2 A45 = pk(fmaf(-a2, px, 1.0f), -py * zi), B45 = pk(-a3, px * zi);
  const f2 NC23 = pk(-1.0f, -py), NC45 = pk(px, 0.0f);     // -c[2..3], -c[4..5]
  const f2 Gp = fma2(bc(c.l), H, G);                        // (gx + l hx, gy + l hy)
  const float gx = lo(Gp), gy = hi(Gp), hx = lo(H), hy = hi(H);
  f2 V0[3], V1[3];
  V0[0] = mul2(Gp, bc(zi));
  V0[1] = fma2(bc(gx), A23, fma2(bc(gy), B23, mul2(bc(c.l), NC23)));
  V0[2] = fma2(bc(gx), A45, fma2(bc(gy), B45, mul2(bc(c.l), NC45)));
  V1[0] = mul2(H, bc(zi));
  V1[1] = fma2(bc(hx), A23, fma2(bc(hy), B23, NC23));
  V1[2] = fma2(bc(hx), A45, fma2(bc(hy), B45, NC45));
  // b -= J^T W r
  stage_b_rank1(acc, V0, wgt * c.wd0, -fmaf(c.l, ez, ei));
  stage_b_rank1(acc, V1, wgt * c.wd1, -ez);
}

// Sum the kNormalValues accumulators of a row over the 32 lanes of its warp in a fixed order (halving exchange: partner
// lane ^ 16, ^ 8, ... ^ 1; 31 shuffles instead of 5 x 28) and store the row's totals: lane l ends up with value l.
__device__ __forceinline__ void flush_row_partial(const StageBAcc& acc, int lane, float* row_out) {
  float a[32];
  stage_b_values(acc, a);
#pragma unroll
  for (int i = kNormalValues; i < 32; ++i) a[i] = 0.f;
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
    const bool up = (lane & half) != 0;
#pragma unroll
    for (int j = 0; j < half; ++j) {
      const float mine = up ? a[half + j] : a[j];
      const float send = up ? a[j] : a[half + j];
      a[j] = mine + __shfl_xor_sync(kFullMask, send, half);
    }
  }
  if (lane < kNormalValues) row_out[lane] = a[0];
}

// optional per-pixel dump of the residual records (dvo_b200_residual_image): seven planes of n floats
struct RecordDump {
  float* planes;   // nullptr: off
  int n;
};
__device__ __noinline__ void dump_record(const RecordDump& dump, size_t i, bool valid, f2 E, f2 G, f2 H, float z) {
  const float nanv = __int_as_float(0x7fc00000);
  float* p = dump.planes + i;
  const size_t n = (size_t)dump.n;
  p[0] = valid ? lo(E) : nanv; p[n] = valid ? hi(E) : nanv;
  p[2 * n] = valid ? lo(G) : nanv; p[3 * n] = valid ? hi(G) : nanv;
  p[4 * n] = valid ? lo(H) : nanv; p[5 * n] = valid ? hi(H) : nanv;
  p[6 * n] = valid ? z : nanv;
}

// Stage B over this CTA's strips.  row_base[y]: number of valid points before row y inside this CTA (only read
// when this CTA holds the tail of the point list); points with rank >= n_keep are the dropped tail of
// computeCompleteDataLogLikelihood (dense_tracking_impl.cpp:413-422).
template <bool kDump>
__device__ __forceinline__ void stage_b_run(TilePipe& tp, const PairLevel& pl, const LevelGeom& g, const StageConsts& c,
                                            const StageBConsts& cb, const int* row_base, const int* strip_base, long long n_keep,
                                            const RecordDump& dump, float* row_partial, unsigned& tile_count, int* error_flag,
                                            PipeTiming& tm) {
  const int lane = threadIdx.x & 31, q = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const int ntiles = g.nmine * g.nbands;
  const unsigned tbase = tile_count;
  tile_count += ntiles;
  if (q == kConsumerWarps) {   // the producer warp
    produce_tiles<true>(tp, pl, g, c, tbase, ntiles, error_flag, tm);
    return;
  }
  int i = 0;
  const unsigned tp_s = pin(smem_u32(&tp));
  const unsigned my_ref = (unsigned)(offsetof(StageBuf, ref0) + (q * kTileW + lane) * 8);
  const unsigned my_tx = (unsigned)(offsetof(StageBuf, tx) + lane * 4);
  const int gw = g.w, gh = g.h, gnb = g.nbands, gpitch = g.pitch;
  for (int sk = 0, s = g.strip0; sk < g.nmine; ++sk, s += g.strip_step) {
    const int y = s * kTileH + q;
    const bool row_ok = y < gh;
    const float ty = __ldg(pl.rtmpl + gw + min(y, gh - 1));
    // the dropped tail of the log-likelihood (points of rank >= n_keep): only the strip(s) that reach past n_keep look at ranks
    const long long sbase = __ldcg(strip_base + s);
    const bool cta_has_tail = (long long)__ldcg(strip_base + s + 1) > n_keep;                 // warp-uniform
    const int keep_rank = (int)max(min(n_keep - sbase, (long long)0x7fffffff), (long long)-1);   // first dropped rank, strip-relative
    int rank = 0;              // rank of the row's first point inside its strip
    if (cta_has_tail && row_ok) rank = __ldcg(row_base + y);
    StageBAcc acc;             // one image row at a time: the row's sums leave the warp in a fixed order (flush_row_partial)
    stage_b_init(acc);
    for (int b = 0; b < gnb; ++b, ++i) {
      const unsigned t = tbase + i;
      const unsigned bufi = t % kStages;
      const int x0 = b * kTileW, bw = min(kTileW, gw - x0);
      const long long tw0 = DVO_CLOCK(tm);
      mbar_wait_s(tp_s + (unsigned)offsetof(TilePipe, full) + bufi * 8u, (t / kStages) & 1u, error_flag);
      DVO_ADD(tm, wait_full_b, DVO_CLOCK(tm) - tw0);
      const unsigned bufs = tp_s + bufi * (unsigned)sizeof(StageBuf);
      const int4 d0 = lds_i4(tp_s + (unsigned)offsetof(TilePipe, desc) + bufi * 32u);
      if (row_ok && !d0.x) {
        const int4 d1 = lds_i4(tp_s + (unsigned)offsetof(TilePipe, desc) + bufi * 32u + 16u);
        const WinView wv = make_view(bufs, d0, d1, pl.c3, gw, gh, gpitch);
        const int nr = (bw + 31) >> 5;
        unsigned refa = bufs + my_ref;
        unsigned txa = bufs + my_tx;
        const int xlim = bw - lane;
#pragma unroll 1
        for (int r = 0; r < nr; ++r, refa += 256, txa += 128) {
          const f2 rz = lds_f2_at(refa);
          const f2 gr = lds_f2<sizeof(float2) * kRecP1>(refa);              // the gradient rows of the record
          const float tx = lds_f32(txa);
          float z = hi(rz);
          if (bw < kTileW) z = (r * 32 < xlim) ? z : __int_as_float(0x7fc00000);
          const PixelProjection p = project_pixel(tx, ty, z, c);
          f2 E, G, H;
          const bool valid = record_pixel(p, wv, lo(rz), z, gr, c, E, G, H);
          DVO_ADD(tm, rounds, 1); DVO_ADD(tm, slow_rounds, wv.exact ? 0 : 1);
          bool keep = valid;
          if (cta_has_tail) {   // warp-uniform
            const unsigned m = __ballot_sync(kFullMask, valid);
            keep = valid && (rank + __popc(m & lt_mask)) < keep_rank;
            rank += __popc(m);
          }
          if (kDump && r * 32 < xlim) dump_record(dump, (size_t)y * gw + x0 + r * 32 + lane, valid, E, G, H, z);
          // rejected points: zero weight and finite stand-ins (their own values may be NaN)
          const float ei = valid ? lo(E) : 0.f, ez = valid ? hi(E) : 0.f;
          const float wall = student_weight(c, ei, ez);
          const float wgt = valid ? wall : 0.f;
          // (tx too: past a partial band it comes from shared memory no copy has written)
          stage_b_pixel(acc, cb, wgt, keep, ei, ez, valid ? G : 0ull, valid ? H : 0ull, valid ? z : 1.0f, valid ? tx : 0.f, ty);
        }
      } else if (kDump && row_ok) {
        for (int xl = lane; xl < bw; xl += 32) dump_record(dump, (size_t)y * gw + x0 + xl, false, 0ull, 0ull, 0ull, 0.f);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive_s(tp_s + (unsigned)offsetof(TilePipe, empty) + bufi * 8u);
    }
    if (row_ok) flush_row_partial(acc, lane, row_partial + (size_t)y * kNormalValues);
  }
}

// flush the product of the pending log-likelihood terms and unpack: out[0] = ll sum,
// out[1..21] = A upper triangle (row-major), out[22..27] = b
__device__ __forceinline__ void stage_b_values(const StageBAcc& acc, float out[]) {
  out[0] = acc.llsum * 0.69314718055994531f;
  out[1] = lo(acc.r0[0]); out[2] = hi(acc.r0[0]); out[3] = lo(acc.r0[1]); out[4] = hi(acc.r0[1]); out[5] = lo(acc.r0[2]); out[6] = hi(acc.r0[2]);
  out[7] = hi(acc.r1[0]); out[8] = lo(acc.r1[1]); out[9] = hi(acc.r1[1]); out[10] = lo(acc.r1[2]); out[11] = hi(acc.r1[2]);
  out[12] = lo(acc.r2[0]); out[13] = hi(acc.r2[0]); out[14] = lo(acc.r2[1]); out[15] = hi(acc.r2[1]);
  out[16] = hi(acc.r3[0]); out[17] = lo(acc.r3[1]); out[18] = hi(acc.r3[1]);
  out[19] = lo(acc.r4); out[20] = hi(acc.r4);
  out[21] = hi(acc.r5);
  out[22] = lo(acc.b[0]); out[23] = hi(acc.b[0]); out[24] = lo(acc.b[1]); out[25] = hi(acc.b[1]); out[26] = lo(acc.b[2]); out[27] = hi(acc.b[2]);
}

__device__ __forceinline__ void load_stage_b_consts(const PairState& st, StageBConsts& c) {
  c.P00 = __ldcg(&st.precision[0]); c.P01 = __ldcg(&st.precision[1]); c.P10 = __ldcg(&st.precision[2]); c.P11 = __ldcg(&st.precision[3]);
  c.l = c.P01 / c.P00;
  c.wd0 = c.P00;
  c.wd1 = c.P11 - c.P01 * c.l;
}

}  // namespace dvo_b200
