// The photometric mode on the CPU oracle (test infrastructure, like the oracle itself): the affine brightness model of
// include/dvo_b200.h ("photometric mode") on top of the oracle's own residual, weight, scale and log-likelihood code, in
// every orc_mode.  The oracle's translation unit is compiled into this one unchanged, so that its internal functions serve
// both; tests/photometric_oracle.py builds the shared library with the oracle's flags (oracle/Makefile).
//
//   residual   the reference intensity of every selected point becomes alpha I_ref + beta before the oracle's residual
//              loop (rounded to nearest; fused_pixel_math: fmaf(alpha, I_ref, beta), else the unfused product and sum),
//              with (alpha, beta) as float.  At (1, 0) that is I_ref exactly, so every mode computes its default residual.
//   normal equations  8 x 8: the oracle's per-entry arithmetic over the Jacobian rows extended by de_i/dalpha = -I_ref/255,
//              de_i/dbeta = -1/255 (intensity row) and zeros (depth row); f32_serial_accum: fp32 in point order (the
//              pose block equals the default FAITHFUL A and b bit for bit), else fp64.
//   match      DenseTracker::match with (alpha, beta) a Revertable updated with the pose: the top of every iteration adds
//              the last accepted increment, a rejected iteration reverts both, levels carry (alpha, beta) over; the
//              information is the Schur complement of the 8 x 8 (mu included) onto the pose.
#include "../../oracle/dvo_oracle.cpp"

namespace {

// Eigen-style pivoted LDL^T of a symmetric n x n (n <= 8): ldlt_solve6's algorithm for any size.
void ldlt_solve_n(const double* Ain, const double* bin, double* x, int n) {
  double A[64];
  std::memcpy(A, Ain, sizeof(double) * n * n);
  int perm[8];
  for (int k = 0; k < n; ++k) {
    int piv = k;
    double best = std::fabs(A[k * n + k]);
    for (int i = k + 1; i < n; ++i)
      if (std::fabs(A[i * n + i]) > best) { best = std::fabs(A[i * n + i]); piv = i; }
    perm[k] = piv;
    if (piv != k) {
      for (int j = 0; j < n; ++j) std::swap(A[k * n + j], A[piv * n + j]);
      for (int i = 0; i < n; ++i) std::swap(A[i * n + k], A[i * n + piv]);
    }
    for (int j = 0; j < k; ++j) A[k * n + k] -= A[k * n + j] * A[k * n + j] * A[j * n + j];
    double d = A[k * n + k];
    for (int i = k + 1; i < n; ++i) {
      double s = A[i * n + k];
      for (int j = 0; j < k; ++j) s -= A[i * n + j] * A[k * n + j] * A[j * n + j];
      A[i * n + k] = (d != 0.0) ? s / d : 0.0;
    }
  }
  double y[8];
  for (int i = 0; i < n; ++i) y[i] = bin[i];
  for (int k = 0; k < n; ++k) std::swap(y[k], y[perm[k]]);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j) y[i] -= A[i * n + j] * y[j];
  double dmax = 0;
  for (int i = 0; i < n; ++i) dmax = std::fmax(dmax, std::fabs(A[i * n + i]));
  double tol = std::fmax(dmax * DBL_EPSILON, 1.0 / DBL_MAX);
  for (int i = 0; i < n; ++i) y[i] = std::fabs(A[i * n + i]) > tol ? y[i] / A[i * n + i] : 0.0;
  for (int i = n - 1; i >= 0; --i)
    for (int j = i + 1; j < n; ++j) y[i] -= A[j * n + i] * y[j];
  for (int k = n - 1; k >= 0; --k) std::swap(y[k], y[perm[k]]);
  for (int i = 0; i < n; ++i) x[i] = y[i];
}

// A_xx - A_xp A_pp^-1 A_px of an 8 x 8 onto its first 6 unknowns, fp64, the 2 x 2 inverse written out
void schur_pose(const double A[64], double S[36]) {
  const double a = A[6 * 8 + 6], c = A[6 * 8 + 7], d = A[7 * 8 + 7];
  const double rdet = 1.0 / (a * d - c * c);
  const double i00 = d * rdet, i01 = -c * rdet, i11 = a * rdet;
  for (int i = 0; i < 6; ++i) {
    const double g0 = i00 * A[i * 8 + 6] + i01 * A[i * 8 + 7], g1 = i01 * A[i * 8 + 6] + i11 * A[i * 8 + 7];
    for (int j = 0; j < 6; ++j) S[i * 6 + j] = A[i * 8 + j] - (g0 * A[j * 8 + 6] + g1 * A[j * 8 + 7]);
  }
}

// the selection with the brightness model applied to the reference intensities
void apply_brightness(std::vector<RefPoint>& pts, const double ab[2], const orc_mode& mode) {
  const float a = float(ab[0]), b = float(ab[1]);
  for (RefPoint& p : pts) p.i = mode.fused_pixel_math ? std::fmaf(a, p.i, b) : a * p.i + b;
}

void normal_equations8(const std::vector<ErrPoint>& e, const std::vector<float>& w, const float P[4], const Level& R,
                       const orc_mode& mode, double A[64], double b[8]) {
  const float wref0 = -1.0f / 255.0f;
  const size_t n = e.size();
  float Af[64] = {0}, bf[8] = {0};
  double Ad[64] = {0}, bd[8] = {0};
  for (size_t k = 0; k < n; ++k) {
    float J0[8], J1[8];
    jacobian_rows<float>(e[k].x, e[k].y, e[k].z, e[k].e[2], e[k].e[3], e[k].e[4], e[k].e[5], J0, J1);
    J0[6] = wref0 * R.ch[0][size_t(e[k].pix)]; J0[7] = wref0;
    J1[6] = 0.0f; J1[7] = 0.0f;
    if (mode.f32_serial_accum) {
      const float W[4] = {w[k] * P[0], w[k] * P[1], w[k] * P[2], w[k] * P[3]};
      const float r0 = e[k].e[0], r1 = e[k].e[1];
      for (int i = 0; i < 8; ++i) {
        const float ua = J0[i] * W[0] + J1[i] * W[2], ub = J0[i] * W[1] + J1[i] * W[3];
        for (int j = i; j < 8; ++j) Af[i * 8 + j] += ua * J0[j] + ub * J1[j];
        bf[i] -= ua * r0 + ub * r1;
      }
    } else {
      const double W[4] = {double(w[k]) * P[0], double(w[k]) * P[1], double(w[k]) * P[2], double(w[k]) * P[3]};
      const double r0 = e[k].e[0], r1 = e[k].e[1];
      for (int i = 0; i < 8; ++i) {
        const double ua = J0[i] * W[0] + J1[i] * W[2], ub = J0[i] * W[1] + J1[i] * W[3];
        for (int j = i; j < 8; ++j) Ad[i * 8 + j] += ua * J0[j] + ub * J1[j];
        bd[i] -= ua * r0 + ub * r1;
      }
    }
  }
  for (int i = 0; i < 8; ++i)
    for (int j = 0; j < 8; ++j) {
      const int u = i <= j ? i * 8 + j : j * 8 + i;
      A[i * 8 + j] = mode.f32_serial_accum ? double(Af[u]) : Ad[u];
    }
  for (int i = 0; i < 8; ++i) b[i] = mode.f32_serial_accum ? double(bf[i]) : bd[i];
}

}  // namespace

extern "C" {

void orc_ldlt_solve8(const double A[64], const double b[8], double x[8]) { ldlt_solve_n(A, b, x, 8); }
void orc_schur_pose(const double A[64], double S[36]) { schur_pose(A, S); }

int64_t orc_residual_image_photometric(const orc_pyramid* ref, const orc_pyramid* cur, int level, const double T[16],
                                       const double ab[2], float ti, float td, const orc_mode* mode, float* planes7) {
  const Level& R = ref->levels[level];
  const Level& C = cur->levels[level];
  std::vector<RefPoint> pts;
  select_points(R, ti, td, pts);
  apply_brightness(pts, ab, *mode);
  LevelConsts c;
  make_level_consts(C, T, c);
  std::vector<ErrPoint> e;
  compute_residuals(pts, C, c, *mode, e);
  const size_t N = size_t(R.w) * R.h;
  for (size_t i = 0; i < 7 * N; ++i) planes7[i] = kNaNf;
  for (const ErrPoint& q : e) {
    for (int k = 0; k < 6; ++k) planes7[size_t(k) * N + q.pix] = q.e[k];
    planes7[6 * N + q.pix] = q.z;
  }
  return int64_t(e.size());
}

int64_t orc_linearize_photometric(const orc_pyramid* ref, const orc_pyramid* cur, int level, const double T[16],
                                  const double ab[2], float ti, float td, int use_weights, const float prev_precision[4],
                                  const orc_mode* mode, float precision_out[4], float* ll_out, double A_out[64],
                                  double b_out[8]) {
  const Level& R = ref->levels[level];
  const Level& C = cur->levels[level];
  std::vector<RefPoint> pts;
  select_points(R, ti, td, pts);
  apply_brightness(pts, ab, *mode);
  LevelConsts c;
  make_level_consts(C, T, c);
  std::vector<ErrPoint> e;
  int64_t n = compute_residuals(pts, C, c, *mode, e);
  if (n < 6) return n;
  std::vector<float> w;
  if (!use_weights) w.assign(size_t(n), 1.0f);
  else compute_weights(e, prev_precision, *mode, w);
  float Cov[4];
  compute_scale(e, w, *mode, Cov);
  inverse2(Cov, precision_out);
  *ll_out = compute_ll(e, precision_out, *mode);
  normal_equations8(e, w, precision_out, R, *mode, A_out, b_out);
  return n;
}

// orc_match in the photometric mode.  ab_init: (alpha, beta) at the start, NULL = (1, 0); ab_out: the final values.
int orc_match_photometric(orc_pyramid* ref, orc_pyramid* cur, const orc_config* cfg, const double T_init[16],
                          const double ab_init[2], const orc_mode* mode_p, orc_result* result, double ab_out[2],
                          orc_iteration_stats* iters, int max_iters, int* num_iters) {
  const orc_mode mode = *mode_p;
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
    double dab[2] = {0.0, 0.0};   // the (alpha, beta) part of the increment the next iteration applies
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
      {
        const AB prev = ab.value;
        ab.update() = AB{{prev.v[0] + dab[0], prev.v[1] + dab[1]}};
      }
      double T[16];
      se3_matrix(estimate.value, T);
      LevelConsts c;
      make_level_consts(C, T, c);
      pts = pts0;
      apply_brightness(pts, ab.value.v, mode);
      int64_t n = compute_residuals(pts, C, c, mode, err);
      it.valid_constraints = n;
      if (n < 6) {
        initial.revert(); estimate.revert(); ab.revert();
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
      double sq = 0;
      for (int i = 0; i < 6; ++i) sq += li[i] * li[i];
      it.prior_log_likelihood = cfg->mu * sq;
      last_error = error;
      error = -double(ll);
      accept = error < last_error;
      if (!accept) {
        initial.revert(); estimate.revert(); ab.revert();
        ls.termination = ORC_TERM_LOG_LIKELIHOOD_DECREASED;
        level_iters.push_back(it);
        break;
      }
      normal_equations8(err, weights, precision, R, mode, A, b);
      for (int i = 0; i < 6; ++i) {
        A[i * 8 + i] += cfg->mu;
        b[i] += cfg->mu * li[i];
      }
      ldlt_solve_n(A, b, x, 8);
      dab[0] = x[6]; dab[1] = x[7];
      for (int i = 0; i < 6; ++i) it.increment[i] = x[i];
      schur_pose(A, it.information);
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
