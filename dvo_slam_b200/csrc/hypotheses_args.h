// hypotheses_args.h -- multi-hypothesis alignment (dvo_b200_match_batch_hypotheses[_modes]): the checks of its arguments that
// need no CUDA call, and the rule that picks one screened hypothesis per pair.  Plain C++ that nvcc also compiles for the
// device, so that both run on the host alone (tests/native/hypotheses_args.cpp, tests/native/hypotheses_modes_args.cpp);
// capi.cu runs the checks before anything is staged, uploaded or launched, and k_pick_hypotheses (tracker.cu) runs the rule.
#pragma once
#include <cstddef>
#include <cstdint>
#include <limits>
#include <string>

#include "../../include/dvo_b200.h"
#include "maps_args.h"
#include "prior_args.h"

#ifndef DVO_HD
#ifdef __CUDACC__
#define DVO_HD __host__ __device__ __forceinline__
#else
#define DVO_HD inline
#endif
#endif

namespace dvo_b200 {

// x is neither infinite nor NaN (x - x is 0 exactly then), without a library call that differs between host and device
DVO_HD bool finite_fp64(double x) { return x - x == 0.0; }

// The score of one screened hypothesis from the dvo_b200_level_stats of its screening level, or NaN if it is not eligible:
// eligible iff it has an iteration with an increment, its constraint ratio last_increment_valid_constraints / valid_pixels
// (ConstraintRatioVoter, in fp64) is >= min_ratio, and the score last_increment_log_likelihood /
// last_increment_valid_constraints (the per-constraint negative log-likelihood; lower is better) is finite.
DVO_HD double hypothesis_score(int has_increment, long long inc_constraints, long long valid_pixels, double inc_log_likelihood,
                               double min_ratio) {
  const double nan = std::numeric_limits<double>::quiet_NaN();
  if (!has_increment) return nan;
  const double ratio = (double)inc_constraints / (double)valid_pixels;
  if (!(ratio >= min_ratio)) return nan;
  const double score = inc_log_likelihood / (double)inc_constraints;
  return finite_fp64(score) ? score : nan;
}

// The hypothesis to continue: the eligible one (score not NaN) with the smallest score, the lowest index on a tie (scan
// upwards, replace on a strict <); 0 if none is eligible.
DVO_HD int pick_hypothesis(const double* scores, int k) {
  int best = -1;
  for (int j = 0; j < k; ++j)
    if (scores[j] == scores[j] && (best < 0 || scores[j] < scores[best])) best = j;
  return best < 0 ? 0 : best;
}

// The checks of dvo_b200_match_batch_hypotheses before those of dvo_b200_match_batch, in this order: a NULL hypotheses,
// results or best; k outside [1, DVO_B200_MAX_HYPOTHESES]; with a cfg, use_initial_estimate 0 and a screen_level outside
// [last_level, first_level]; a min_constraint_ratio that is not finite or lies outside [0, 1]; then, for n > 0, each
// hypothesis: a non-finite entry or a bottom row other than (0, 0, 0, 1).  A NULL cfg or n <= 0 is left to the batch checks
// that follow.  Returns "" or the message, prefixed with "match_batch_hypotheses: ".
inline std::string hypotheses_args_error(const dvo_b200_config* cfg, int32_t n, int32_t k, const double* hypotheses,
                                         int32_t screen_level, double min_constraint_ratio, const void* results,
                                         const int32_t* best) {
  const std::string fn = "match_batch_hypotheses: ";
  if (!hypotheses) return fn + "hypotheses is null";
  if (!results) return fn + "results is null";
  if (!best) return fn + "best is null";
  if (k < 1 || k > DVO_B200_MAX_HYPOTHESES)
    return fn + "k = " + std::to_string(k) + " outside [1, " + std::to_string(DVO_B200_MAX_HYPOTHESES) + "]";
  if (cfg) {
    if (!cfg->use_initial_estimate) return fn + "cfg->use_initial_estimate must be 1: the hypotheses are the initial estimates";
    if (screen_level < cfg->last_level || screen_level > cfg->first_level)
      return fn + "screen_level = " + std::to_string(screen_level) + " outside [last_level, first_level] = [" +
             std::to_string(cfg->last_level) + ", " + std::to_string(cfg->first_level) + "]";
  }
  if (!finite_fp64(min_constraint_ratio) || min_constraint_ratio < 0.0 || min_constraint_ratio > 1.0)
    return fn + "min_constraint_ratio is not a finite value in [0, 1]";
  for (int64_t h = 0; h < (int64_t)n * k; ++h) {
    const double* T = hypotheses + (size_t)h * 16;
    const std::string which = "hypothesis " + std::to_string(h % k) + " of pair " + std::to_string(h / k);
    for (int i = 0; i < 16; ++i)
      if (!finite_fp64(T[i])) return fn + which + " is not finite";
    if (T[12] != 0.0 || T[13] != 0.0 || T[14] != 0.0 || T[15] != 1.0) return fn + which + " has a bottom row other than (0, 0, 0, 1)";
  }
  return "";
}

// The checks of dvo_b200_match_batch_hypotheses_modes, in this order: those of hypotheses_args_error; photometric_init without
// photometric; screen_photometric without photometric; with a prior, cfg->mu != 0, then each hypothesis's Lambda
// (prior_matrix_error; skipped with a NULL cfg); each hypothesis's (alpha, beta)_0 not finite; with maps, everything maps_args_error refuses, at the
// batch's largest extents `extent` (NULL: the batch checks that follow will refuse the batch, so the maps are checked as
// for n = 0).  A NULL cfg or n <= 0 is left to the batch checks.  Every message is prefixed with "match_batch_hypotheses: ",
// and the per-hypothesis ones name the hypothesis as hypotheses_args_error does.
template <typename Where>
std::string hypotheses_modes_args_error(const dvo_b200_config* cfg, int32_t n, int32_t k, const double* hypotheses, int32_t screen_level,
                                        double min_constraint_ratio, const void* results, const int32_t* best,
                                        const double* prior_information, const double* photometric_init, const double* photometric,
                                        const double* screen_photometric, const dvo_b200_weight_maps* maps, const MapsExtent* extent,
                                        int device, Where where) {
  const std::string why = hypotheses_args_error(cfg, n, k, hypotheses, screen_level, min_constraint_ratio, results, best);
  if (!why.empty()) return why;
  const std::string fn = "match_batch_hypotheses: ";
  if (photometric_init && !photometric) return fn + "photometric_init without photometric";
  if (screen_photometric && !photometric) return fn + "screen_photometric without photometric";
  auto which = [&](int64_t h) { return "hypothesis " + std::to_string(h % k) + " of pair " + std::to_string(h / k); };
  if (prior_information && cfg) {
    if (cfg->mu != 0.0) return fn + "cfg->mu must be 0: the prior replaces mu I";
    for (int64_t h = 0; h < (int64_t)n * k; ++h) {
      const std::string bad = prior_matrix_error(prior_information + (size_t)h * 36);
      if (!bad.empty()) return fn + "prior_information of " + which(h) + " " + bad;
    }
  }
  if (photometric_init)
    for (int64_t h = 0; h < (int64_t)n * k; ++h)
      if (!finite_fp64(photometric_init[2 * h]) || !finite_fp64(photometric_init[2 * h + 1]))
        return fn + "photometric_init of " + which(h) + " is not finite";
  if (maps) {
    const std::string bad = maps_args_error(maps, extent ? n : 0, extent ? *extent : MapsExtent{0, 0, 0, 0}, device, where);
    const std::string maps_fn = "match_batch_maps: ";
    if (!bad.empty()) return fn + bad.substr(maps_fn.size());
  }
  return "";
}

}  // namespace dvo_b200
