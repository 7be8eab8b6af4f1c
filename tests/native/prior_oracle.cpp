// The motion prior on the CPU oracle (test infrastructure, like the oracle itself): include/dvo_b200.h ("motion prior") on
// top of the oracle's match loop, in every orc_mode and in both the default and the photometric mode.  The photometric
// oracle's translation unit, and through it the oracle's, is compiled into this one unchanged, so that their internal
// functions serve all three; tests/prior_oracle.py builds the shared library with the oracle's flags (oracle/Makefile).
//
//   prior   Lambda (6 x 6, row-major) in place of mu I: s_i = sum_j Lambda_ij li_j in order j = 0..5 from 0, then
//           A_ij += Lambda_ij and b_i += s_i on the pose block, and the prior log-likelihood sum_i li_i s_i.  Built with
//           -ffp-contract=off, so that with Lambda = mu I every term but mu li_i is an exact zero and b_i + s_i is the oracle's
//           unfused b_i + mu li_i.  Everything else is orc_match / orc_match_photometric.
#include "photometric_oracle.cpp"

namespace {

struct PriorTerms {
  double s[6];   // Lambda li
  double ll;     // li^T Lambda li
};

PriorTerms prior_terms(const double L[36], const double li[6]) {
  PriorTerms t;
  t.ll = 0.0;
  for (int i = 0; i < 6; ++i) {
    double s = 0.0;
    for (int j = 0; j < 6; ++j) s += L[i * 6 + j] * li[j];
    t.s[i] = s;
  }
  for (int i = 0; i < 6; ++i) t.ll += li[i] * t.s[i];
  return t;
}

}  // namespace

extern "C" {

// orc_match with a prior information Lambda (36 doubles) in place of cfg->mu I (cfg->mu is ignored).  ab_out == NULL: the
// default 6-unknown mode; else the photometric mode from ab_init (NULL = (1, 0)), the final (alpha, beta) to ab_out.
int orc_match_prior(orc_pyramid* ref, orc_pyramid* cur, const orc_config* cfg, const double T_init[16], const double L[36],
                    const double ab_init[2], const orc_mode* mode_p, orc_result* result, double ab_out[2],
                    orc_iteration_stats* iters, int max_iters, int* num_iters) {
  const orc_mode mode = *mode_p;
  const bool photometric = ab_out != nullptr;
  const int nu = photometric ? 8 : 6;
  int iter_count = 0;
  std::memset(result, 0, sizeof(*result));
  SE3 inc;
  if (cfg->use_initial_estimate) inc = se3_from_matrix(T_init);
  Revertable<SE3> initial{inc, inc};
  Revertable<SE3> estimate{SE3(), SE3()};
  struct AB { double v[2]; };
  Revertable<AB> ab{{{1.0, 0.0}}, {{1.0, 0.0}}};
  if (ab_init) { ab.value.v[0] = ab.old.v[0] = ab_init[0]; ab.value.v[1] = ab.old.v[1] = ab_init[1]; }
  bool accept = true;
  float precision[4] = {0, 0, 0, 0};
  std::vector<RefPoint> pts0, pts;
  std::vector<ErrPoint> err;
  std::vector<float> weights;
  std::vector<orc_iteration_stats> level_iters;

  for (int level = cfg->first_level; level >= cfg->last_level; --level) {
    orc_level_stats& ls = result->levels[result->num_levels++];
    level_iters.clear();
    precision[0] = precision[1] = precision[2] = precision[3] = 0;
    int iteration = 0;
    double error = std::numeric_limits<double>::max(), last_error;
    const Level& C = cur->levels[level];
    const Level& R = ref->levels[level];
    select_points(R, cfg->intensity_derivative_threshold, cfg->depth_derivative_threshold, pts0);
    ls.id = level;
    ls.max_valid_pixels = max_points(ref, level);
    ls.valid_pixels = int64_t(pts0.size());
    ls.termination = -1;
    double A[64], b[8], x[8];
    se3_log(inc, x);
    double dab[2] = {0.0, 0.0};
    do {
      orc_iteration_stats it;
      std::memset(&it, 0, sizeof(it));
      for (int i = 0; i < 36; ++i) it.information[i] = kNaN;
      for (int i = 0; i < 6; ++i) it.increment[i] = kNaN;
      it.level = level;
      it.id = iteration;
      inc = se3_exp(x);
      initial.update() = se3_mul(se3_inverse(inc), initial.value);
      estimate.update() = se3_mul(inc, estimate.value);
      if (photometric) {
        const AB prev = ab.value;
        ab.update() = AB{{prev.v[0] + dab[0], prev.v[1] + dab[1]}};
      }
      double T[16];
      se3_matrix(estimate.value, T);
      LevelConsts c;
      make_level_consts(C, T, c);
      pts = pts0;
      if (photometric) apply_brightness(pts, ab.value.v, mode);
      int64_t n = compute_residuals(pts, C, c, mode, err);
      it.valid_constraints = n;
      if (n < 6) {
        initial.revert(); estimate.revert();
        if (photometric) ab.revert();
        ls.termination = ORC_TERM_TOO_FEW_CONSTRAINTS;
        level_iters.push_back(it);
        break;
      }
      if (iteration == 0) weights.assign(size_t(n), 1.0f);
      else compute_weights(err, precision, mode, weights);
      float Cov[4];
      compute_scale(err, weights, mode, Cov);
      inverse2(Cov, precision);
      float ll = compute_ll(err, precision, mode);
      it.tdist_log_likelihood = -double(ll);
      for (int i = 0; i < 4; ++i) it.tdist_precision[i] = double(precision[i]);
      double li[6];
      se3_log(initial.value, li);
      const PriorTerms pt = prior_terms(L, li);
      it.prior_log_likelihood = pt.ll;
      last_error = error;
      error = -double(ll);
      accept = error < last_error;
      if (!accept) {
        initial.revert(); estimate.revert();
        if (photometric) ab.revert();
        ls.termination = ORC_TERM_LOG_LIKELIHOOD_DECREASED;
        level_iters.push_back(it);
        break;
      }
      if (photometric) normal_equations8(err, weights, precision, R, mode, A, b);
      else normal_equations(err, weights, precision, mode, A, b);
      for (int i = 0; i < 6; ++i) {
        for (int j = 0; j < 6; ++j) A[i * nu + j] += L[i * 6 + j];
        b[i] += pt.s[i];
      }
      if (photometric) {
        ldlt_solve_n(A, b, x, 8);
        dab[0] = x[6]; dab[1] = x[7];
        schur_pose(A, it.information);
      } else {
        ldlt_solve6(A, b, x);
        for (int i = 0; i < 36; ++i) it.information[i] = A[i];
      }
      for (int i = 0; i < 6; ++i) it.increment[i] = x[i];
      level_iters.push_back(it);
      iteration++;
    } while (accept && linf6(x) > cfg->precision && !(iteration >= cfg->max_iterations_per_level));
    if (linf6(x) <= cfg->precision) ls.termination = ORC_TERM_INCREMENT_TOO_SMALL;
    if (iteration >= cfg->max_iterations_per_level) ls.termination = ORC_TERM_ITERATIONS_EXCEEDED;
    ls.num_iterations = int32_t(level_iters.size());
    for (const orc_iteration_stats& it : level_iters) {
      if (iters && iter_count < max_iters) iters[iter_count] = it;
      iter_count++;
    }
  }
  const orc_level_stats& last_level = result->levels[result->num_levels - 1];
  int pick = last_level.termination != ORC_TERM_LOG_LIKELIHOOD_DECREASED ? int(level_iters.size()) - 1
                                                                          : int(level_iters.size()) - 2;
  double Tm[16];
  se3_matrix(se3_inverse(estimate.value), Tm);
  std::memcpy(result->transformation, Tm, sizeof(Tm));
  if (pick >= 0) {
    for (int i = 0; i < 36; ++i) result->information[i] = level_iters[pick].information[i] * 0.008 * 0.008;
    result->log_likelihood = level_iters[pick].tdist_log_likelihood + level_iters[pick].prior_log_likelihood;
  } else {
    for (int i = 0; i < 36; ++i) result->information[i] = kNaN;
    result->log_likelihood = kNaN;
  }
  if (ab_out) { ab_out[0] = ab.value.v[0]; ab_out[1] = ab.value.v[1]; }
  if (num_iters) *num_iters = iter_count;
  return 0;
}

}  // extern "C"
