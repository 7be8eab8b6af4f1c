// launch_plan.h -- how one match call spreads the pyramid levels of its batch over the persistent level kernel: which
// launches, the segments of each launch, their squad sizes and the pairs each segment hands out.  Plain C++ without CUDA,
// so that the plan can be built and checked on the host alone (tests/native/launch_plan.cpp).
#pragma once
#include <algorithm>
#include <cstdio>
#include <cstdlib>

#include "../../include/dvo_b200.h"

namespace dvo_b200 {

constexpr int kMaxSeg = 4;   // segments of one launch: the coarse levels, then up to three slices of the fine levels

// Developer overrides of the plan (experiments).  They change speed only: every plan returns the same bits.
struct PlanKnobs {
  bool no_walk = false;        // DVO_B200_NO_WALK: one launch per level at every batch size
  bool no_fuse = false;        // DVO_B200_NO_FUSE: the coarse and the fine group in launches of their own
  bool contiguous = false;     // DVO_B200_CONTIGUOUS: CTA r of a squad takes a contiguous range of strips
  int coarse_tiles = 110;      // DVO_B200_COARSE_TILES: levels up to 320x240 (105 tiles) run with one CTA per pair
  bool tail = false;           // DVO_B200_TAIL = "c2,c3": pairs of the 2g and 4g slices of a fused launch
  int tail_pairs[2] = {0, 0};
  int strips_per_cta = 0;      // DVO_B200_STRIPS_PER_CTA: squad size of a level with this many strips per CTA (0: cost model)
  int fine_g = 0;              // DVO_B200_FINE_G: squad size of the non-coarse groups (0: the plan's)
};

// Read on every call, so that a process can change them between calls.
inline PlanKnobs plan_knobs_from_env() {
  PlanKnobs k;
  k.no_walk = getenv("DVO_B200_NO_WALK") != nullptr;
  k.no_fuse = getenv("DVO_B200_NO_FUSE") != nullptr;
  k.contiguous = getenv("DVO_B200_CONTIGUOUS") != nullptr;
  if (const char* e = getenv("DVO_B200_COARSE_TILES")) k.coarse_tiles = atoi(e);
  if (const char* e = getenv("DVO_B200_TAIL")) k.tail = sscanf(e, "%d,%d", &k.tail_pairs[0], &k.tail_pairs[1]) >= 1;
  if (const char* e = getenv("DVO_B200_STRIPS_PER_CTA")) k.strips_per_cta = atoi(e);
  if (const char* e = getenv("DVO_B200_FINE_G")) k.fine_g = atoi(e);
  return k;
}

struct LevelShape { int h, nbands, nstrips; };   // rows, tile columns and strips (tile rows) of one pyramid level

// A group of consecutive pyramid levels that a squad of g CTAs walks a pair through, coarse to fine.
struct PlanSegment {
  int first_li, nlev;          // levels [first_li, first_li + nlev) of the match (index 0 = coarsest)
  int g;                       // CTAs per squad
  int nsquads;                 // squads in the grid
  int strips_per_cta[DVO_B200_MAX_LEVELS];
  int pair_begin, npairs;      // the pairs this segment's queue hands out (a slice of the batch for the fine segments of a fused launch)
  int hmax;                    // rows of the segment's tallest level: the per-squad scratch is sized for it
  int cyclic;                  // 1: CTA r of a squad takes strips r, r + g, ...; 0: contiguous ranges of strips_per_cta strips
};
struct PlanLaunch {
  int nseg;
  PlanSegment seg[kMaxSeg];
};
struct LaunchPlan {
  int nlaunch;
  PlanLaunch launch[DVO_B200_MAX_LEVELS];
};

// Squad size for one level on its own.  A squad of g CTAs gives each CTA spc = ceil(nstrips / g) strips.  Small squads keep
// many pairs in flight and amortise the two barriers and the serial P_k / solve sections of an iteration over more tiles
// per CTA; but the batch is processed in waves of nsquads pairs, and a last wave that is mostly empty wastes more than
// that.  Pairs are handed out from a queue, so a level takes about (pairs per squad + tail) x time per pair, where the
// tail (pairs that need two or three times the mean number of iterations) is worth a bit more than one pair and the time
// per pair goes with (tiles per CTA + per-iteration overhead in tile units).
inline int level_squad_size(int nstrips, int nbands, int grid, int npairs, int forced_spc) {
  // per stage: squad barrier + serial step + pipeline fill, in tile-times.  Fitted on an H100 at batch 512 (DESIGN §6): level 0
  // with g = 2 is 1.3 % faster than g = 3, g = 1 and g >= 4 are slower; the model picks g = 2 there for 43 .. 100.
  const double overhead_tiles = 45.0;
  int best_g = 1;
  double best_cost = -1.0;
  for (int spc = 1; spc <= nstrips; ++spc) {
    const int g = (nstrips + spc - 1) / spc;
    if (g > grid) continue;
    if (spc > 1 && (nstrips + spc - 2) / (spc - 1) == g) continue;   // same g as the previous spc: more work per CTA, nothing gained
    const int nsquads = std::min(grid / g, std::max(npairs, 1));
    const double per_squad = (double)npairs / nsquads;
    double cost = (std::max(per_squad, 1.0) + (npairs > nsquads ? 1.2 : 0.0)) * ((double)spc * nbands + overhead_tiles);
    if (forced_spc > 0) cost = std::abs(spc - forced_spc);
    if (best_cost < 0 || cost < best_cost - 1e-9) { best_cost = cost; best_g = g; }
  }
  return best_g;
}

// The plan of a match over the pyramid levels first .. last (shape: indexed by pyramid level) of npairs pairs on a grid of
// `grid` CTAs.
//
// Levels small enough for one CTA per pair (no squad barriers at all) form one group: a CTA takes a pair from the queue and
// runs it through all of them, so a pair that needs many iterations on one coarse level delays nobody.  The remaining
// (fine) levels form a second group with the squad size of the finest level; a squad likewise walks its pair through both.
// With few pairs every level gets its own launch and the squad size that minimises its latency.
//
// A coarse group (one CTA per pair) followed by a fine group runs as ONE launch of several segments: no grid-wide barrier
// and no launch boundary between them, so the CTAs that run out of coarse pairs start on fine pairs while the long coarse
// pairs are still iterating.  The fine group is cut into up to three slices of the pair index with squads of g, 2g and 4g
// CTAs.  Pairs come off a queue, so with one squad size the launch ends with most squads idle while a few finish pairs
// that need two or three times the mean number of iterations.  The last pairs of the batch, which also leave the coarse
// segment last, therefore go to wider squads that finish a pair in a half / a quarter of the time; the slice a pair
// belongs to is fixed by its index, so results do not depend on timing.
inline LaunchPlan make_launch_plan(const LevelShape* shape, int first, int last, int grid, int npairs, const PlanKnobs& knobs) {
  const int nlev = first - last + 1;
  auto level = [&](int li) -> const LevelShape& { return shape[first - li]; };
  auto coarse = [&](int li) { return level(li).nstrips * level(li).nbands <= knobs.coarse_tiles; };
  auto segment = [&](int first_li, int nl, int g, int pair_begin, int np) {
    PlanSegment S{};
    S.first_li = first_li; S.nlev = nl; S.g = g;
    S.nsquads = std::min(grid / g, std::max(np, 1));
    S.pair_begin = pair_begin; S.npairs = np;
    for (int k = 0; k < nl; ++k) {
      const LevelShape& L = level(first_li + k);
      const int g_eff = std::min(g, L.nstrips);
      S.strips_per_cta[k] = (L.nstrips + g_eff - 1) / g_eff;
      S.hmax = std::max(S.hmax, L.h);
    }
    S.cyclic = knobs.contiguous ? 0 : 1;
    return S;
  };

  PlanSegment groups[DVO_B200_MAX_LEVELS];
  int ngroups = 0;
  const bool walk = npairs >= grid / 4 && !knobs.no_walk;
  for (int li = 0; li < nlev;) {
    int nl = 1;
    int g = level_squad_size(level(li).nstrips, level(li).nbands, grid, npairs, knobs.strips_per_cta);
    if (walk) {
      if (coarse(li)) g = 1;
      for (; li + nl < nlev && coarse(li + nl) == coarse(li); ++nl)   // the finest level of a fine group decides
        if (!coarse(li)) g = level_squad_size(level(li + nl).nstrips, level(li + nl).nbands, grid, npairs, knobs.strips_per_cta);
    }
    if (knobs.fine_g > 0 && !coarse(li)) g = std::min(knobs.fine_g, grid);
    groups[ngroups++] = segment(li, nl, g, 0, npairs);
    li += nl;
  }

  LaunchPlan plan{};
  if (!(ngroups == 2 && groups[0].g == 1 && !knobs.no_fuse)) {
    for (int gi = 0; gi < ngroups; ++gi) {
      PlanLaunch& L = plan.launch[plan.nlaunch++];
      L.nseg = 1; L.seg[0] = groups[gi];
    }
    return plan;
  }
  PlanLaunch& L = plan.launch[plan.nlaunch++];
  L.seg[L.nseg++] = groups[0];
  const PlanSegment& F = groups[1];
  int min_strips = 1 << 30;
  for (int k = 0; k < F.nlev; ++k) min_strips = std::min(min_strips, level(F.first_li + k).nstrips);
  const int g2 = 2 * F.g, g3 = 4 * F.g;
  const bool fit2 = g2 <= min_strips && g2 <= grid, fit3 = g3 <= min_strips && g3 <= grid;
  int c2 = fit2 ? (int)(1.8 * (grid / g2) + 0.5) : 0;
  int c3 = c2 && fit3 ? (int)(1.8 * (grid / g3) + 0.5) : 0;
  if (knobs.tail) { c2 = fit2 ? knobs.tail_pairs[0] : 0; c3 = c2 && fit3 ? knobs.tail_pairs[1] : 0; }
  const int keep = 2 * (grid / F.g);                     // the first slice keeps at least two pairs per squad
  if (npairs - c2 - c3 < keep) c3 = 0;
  if (npairs - c2 < keep) c2 = 0;
  const int counts[3] = {npairs - c2 - c3, c2, c3};
  for (int k = 0, begin = 0; k < 3; ++k) {
    if (counts[k] <= 0) continue;
    L.seg[L.nseg++] = segment(F.first_li, F.nlev, F.g << k, begin, counts[k]);
    begin += counts[k];
  }
  return plan;
}

}  // namespace dvo_b200
