// tracker.cu -- dvo::DenseTracker::match() (dvo_core/src/dense_tracking.cpp:131-376) for a batch of
// independent frame pairs, all state on the device.
//
// Per Gauss-Newton iteration the reference makes five passes over the points
// (computeResidualsSse, computeWeightsSse, computeScaleSse, computeCompleteDataLogLikelihood and the
// normal-equation loop, dense_tracking.cpp:271-343).  Precision P_k is a global reduction that the
// log-likelihood and J^T W J depend on, so there are exactly two data-parallel stages (stages.cuh):
//   stage A: warp/interpolate/residual/occlusion test, Student-t weight from P_{k-1}, pairwise scale sums
//   stage B: the same residuals again plus gradients, log-likelihood terms and the 21+6 normal-equation
//            coefficients with W = w*P_k
// each followed by a small per-pair step (pair_mid_warp: P_k; pair_end_cta: accept test, 6x6 LDL^T
// solve, SE(3) update, termination logic).  Both stages read their inputs from shared-memory tiles that a
// producer warp fills with bulk asynchronous copies (TMA unit) through an mbarrier pipeline; nothing but
// per-row / per-strip summaries is written.  A batch that fills the GPU runs ALL levels inside ONE persistent
// cooperative launch (k_level_persistent: a coarse segment with one CTA per pair, then slices of the fine levels
// with squads of g, 2g and 4g CTAs); small batches use one launch per level; the test hooks (residual image,
// linearize) run the same kernel for one pair and one iteration.  All sums above an image row are taken in an
// order fixed by the level's geometry, so every plan returns the same bits.
#include "common.cuh"
#include "stages.cuh"
#include "launch_plan.h"
#include "hypotheses_args.h"

#include <cstdio>
#include <cstring>
#include <limits>
#include <cmath>
#include <cstdlib>
#include <algorithm>
#include <type_traits>

namespace dvo_b200 {

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int kEndWarps = 4;   // warps that sum the level's strip partials in pair_end_cta

struct LevelLaunch {
  int w, h, n, pitch;
  int nbands, nstrips;
  int level_index;   // position in Result.Statistics.Levels
  int level_id;      // pyramid level
  int max_iterations;
  int first_level;   // 1 for the coarsest level of the match
  int use_initial_estimate;
  double precision, mu;
};

// ------------------------------------------------------------------------------------------------
// per-pair helpers
// ------------------------------------------------------------------------------------------------
__device__ void prepare_iteration(PairState& st, const PairLevel& pl) {
  // dense_tracking.cpp:259-263
  st.inc = se3_exp(st.x);
  st.initial_old = st.initial;
  st.initial = se3_mul(se3_inverse(st.inc), st.initial);
  st.estimate_old = st.estimate;
  st.estimate = se3_mul(st.inc, st.estimate);
  double T[16];
  se3_matrix(st.estimate, T);
  kt_of(T, pl, st.kt);
}

__device__ void log_iteration(dvo_b200_iteration_stats* ilog, int max_log, int pair, PairState& st, int it_id, int level_id,
                              bool with_increment) {
  if (!ilog || st.iter_log_count >= max_log) { st.iter_log_count++; return; }
  dvo_b200_iteration_stats& e = ilog[(size_t)pair * max_log + st.iter_log_count++];
  e.level = level_id;
  e.id = it_id;
  e.valid_constraints = st.n;
  e.tdist_log_likelihood = st.nll_cur;
  for (int i = 0; i < 4; ++i) e.tdist_precision[i] = (double)st.precision[i];
  e.prior_log_likelihood = st.prior_cur;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (int i = 0; i < 6; ++i) e.increment[i] = with_increment ? st.x[i] : nan;
  for (int i = 0; i < 36; ++i) e.information[i] = with_increment ? st.A_done[i] : nan;
}

// Start of a pyramid level for one pair (dense_tracking.cpp:137-150, 205-210, 238): run by one thread of the squad that
// owns the pair, before the level's first iteration.
__device__ void level_begin(PairState& st, const PairLevel& pl, const double* T_init, int pair, const LevelLaunch& lp) {
  if (lp.first_level) {
    // dense_tracking.cpp:137-150: first increment is the given guess
    st.inc = (lp.use_initial_estimate && T_init) ? se3_from_matrix(T_init + (size_t)pair * 16) : se3_identity();
    st.initial = st.inc; st.initial_old = st.inc;
    st.estimate = se3_identity(); st.estimate_old = se3_identity();
    st.num_levels = 0; st.num_iterations_total = 0; st.iter_log_count = 0;
  }
  // dense_tracking.cpp:205-210
  st.precision[0] = st.precision[1] = st.precision[2] = st.precision[3] = 0.f;
  st.iteration = 0;
  st.error = 1.7976931348623157e308;
  st.last_error = st.error;
  st.have_done = 0;
  st.termination = -1;
  st.level_active = 1;
  st.phase_ok = 0;
  LevelSummary& ls = st.levels[lp.level_index];
  ls.id = lp.level_id; ls.termination = -1;
  ls.max_valid_pixels = pl.max_valid_pixels;
  ls.valid_pixels = pl.rsel[0];
  ls.num_iterations = 0; ls.has_inc = 0; ls.last_n = 0; ls.last_inc_n = -1;
  ls.last_inc_nll = __longlong_as_double(0x7ff8000000000000LL);
  st.num_levels = lp.level_index + 1;
  se3_log(st.inc, st.x);  // dense_tracking.cpp:238
  prepare_iteration(st, pl);
}

// The pair descriptors of all levels and the initial estimates are written by the host into pinned memory; this kernel
// reads them over PCIe (unified addressing) into device memory, which keeps the upload off the H2D copy engine, where it
// would queue behind a bulk image upload of another context.
__global__ void k_stage_words(const uint4* __restrict__ src, uint4* __restrict__ dst, size_t n16) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n16) dst[i] = src[i];
}

// one warp per pair: combine the strip summaries of the level in order -> covariance -> P_k (dense_tracking.cpp:276-295).
// e: the level's nstrips strip summaries; strip_base: nstrips + 1 exclusive prefixes of their valid counts (output).
// kCorrected: the summaries hold the plain sum of w r r^T (no pairing, no odd tail term) and every point is kept.
template <bool kCorrected>
__device__ __noinline__ void pair_mid_warp(PairState& st, int pair, const double* e, int* strip_base, int nstrips,
                                           const LevelLaunch& lp, dvo_b200_iteration_stats* ilog, int max_log, SegCombineSmem& sm) {
  const int lane = threadIdx.x & 31;
  const SegT<double> all = combine_strip_exports_warp(e, nstrips, strip_base, sm);
  if (lane == 0) {
    long long n = all.n;
    st.n = n;
    st.n_keep = kCorrected ? n : (n / 50) * 50;
    LevelSummary& ls = st.levels[lp.level_index];
    ls.num_iterations += 1;   // level_stats.Iterations.push_back (dense_tracking.cpp:249)
    ls.last_n = n;
    st.num_iterations_total += 1;
    if (n < 6) {
      // dense_tracking.cpp:276-284
      st.initial = st.initial_old; st.estimate = st.estimate_old;
      st.termination = DVO_B200_TERM_TOO_FEW_CONSTRAINTS;
      st.phase_ok = 0;
      // the reference's entry is value-initialised apart from ValidConstraints: log-likelihoods and precision are 0
      st.nll_cur = 0; st.prior_cur = 0;
      for (int i = 0; i < 4; ++i) st.precision[i] = 0.f;
      // and no normal equations: what the linearisation hook reports for this iteration (the end step never runs)
      st.ll = 0.f;
      for (int i = 0; i < 36; ++i) st.A[i] = 0.0;
      for (int i = 0; i < 6; ++i) st.b[i] = 0.0;
      log_iteration(ilog, max_log, pair, st, st.iteration, lp.level_id, false);
      // post-loop checks of dense_tracking.cpp:359-363 still apply
      double m = 0; bool nanx = false;
      for (int i = 0; i < 6; ++i) { m = fmax(m, fabs(st.x[i])); nanx |= st.x[i] != st.x[i]; }
      if (!nanx && m <= lp.precision) st.termination = DVO_B200_TERM_INCREMENT_TOO_SMALL;
      if (st.iteration >= lp.max_iterations) st.termination = DVO_B200_TERM_ITERATIONS_EXCEEDED;
      ls.termination = st.termination;
      ls.has_inc = ls.num_iterations >= 2;   // HasIterationWithIncrement (dense_tracking_config.cpp:138-143)
      if (st.termination != DVO_B200_TERM_TOO_FEW_CONSTRAINTS) ls.has_inc = ls.num_iterations >= 1;
      // LastIterationWithIncrement is Iterations.back() for every termination but LogLikelihoodDecreased: this entry
      if (ls.has_inc) { ls.last_inc_n = n; ls.last_inc_nll = 0.0; }
      st.have_done = (st.termination == DVO_B200_TERM_TOO_FEW_CONSTRAINTS) ? -1 : st.have_done;
      st.level_active = 0;
    } else {
      // tail term for odd n, normaliser 1/(n-3) (dense_tracking_impl.cpp:596), symmetric 2x2
      double c[3];
      const bool tail = !kCorrected && ((n - 1) & 1) == 0;
      double s = 1.0 / (double)(n - 3);
      for (int k = 0; k < 3; ++k) c[k] = (all.S0[k] + (tail ? all.wl * all.ol[k] : 0.0)) * s;
      float C0 = (float)c[0], C1 = (float)c[1], C3 = (float)c[2];
      // precision = covariance.inverse() (Eigen 2x2 inverse, dense_tracking.cpp:295), float, unfused
      float det = __fsub_rn(__fmul_rn(C0, C3), __fmul_rn(C1, C1));
      float invdet = __fdiv_rn(1.0f, det);
      for (int i = 0; i < 4; ++i) st.precision_prev[i] = st.precision[i];
      st.precision[0] = __fmul_rn(C3, invdet);
      st.precision[1] = __fmul_rn(-C1, invdet);
      st.precision[2] = __fmul_rn(-C1, invdet);
      st.precision[3] = __fmul_rn(C0, invdet);
      st.phase_ok = 1;
    }
  }
  __syncwarp();
}

// End of an iteration (dense_tracking.cpp:297-363): add the level's strip partials, log-likelihood, accept test, solve,
// pose update, termination.  Every thread of the CTA calls; thread 0 does the scalar part in two steps:
//   critical : everything the other CTAs of the squad wait for -- the new K*T and iteration flag, or
//              level_active = 0 -- followed by `release` (the squad barrier of the persistent kernel);
//   deferred : Revertable bookkeeping, statistics, the iteration log.  It finishes before this CTA arrives at
//              the squad's next barrier, so the next P_k / end step (run by whichever CTA arrives last) sees it.
struct PairEndSmem {
  static constexpr bool kAffine = false;
  static constexpr bool kPrior = false;
  double part[kEndWarps][32];
};
// The photometric mode: 45 values per strip, and the pair's brightness state (set by the kernel before the call).  They
// travel in the end step's shared block rather than as arguments: an extra argument of the __noinline__ pair_end_cta would
// change the call sequence, and with it the code, of the default instances.
struct PairEndSmemAffine {
  static constexpr bool kAffine = true;
  static constexpr bool kPrior = false;
  double part[kEndWarps][64];
  AffineState* aff;
  int keep_system;   // 1: the linearisation hook, which reads the 8 x 8 system back (AffineState::A, b)
};
// A motion prior (dvo_b200_match_batch_prior): the pair's 6 x 6 information Lambda in place of mu I.  The kernel sets `prior`
// (PersistentArgs::prior) once at its start; in the end step warp kEndWarps, idle while warps 0 .. kEndWarps-1 sum the strip
// partials, copies the pair's Lambda into `lam`, and the barrier after the partial sums orders it before thread 0 reads it,
// so its loads stay off the critical path.
template <typename Base>
struct PairEndSmemPrior : Base {
  static constexpr bool kPrior = true;
  const double* prior;
  double lam[36];
};

// Lambda (row-major) on the pose block of the n x n system A x = b at log(initial) = li: A_ij += Lambda_ij, and
// b_i += sum_j Lambda_ij li_j as an in-order FMA chain.  With Lambda = mu I every added term but mu li_i is an exact zero,
// so this is the default path's A_ii + mu and fma(mu, li_i, b_i) bit for bit.
template <int kN>
__device__ __forceinline__ void add_prior(const double lam[36], const double li[6], double* A, double* b) {
  for (int i = 0; i < 6; ++i) {
    double bi = b[i];
    for (int j = 0; j < 6; ++j) { A[i * kN + j] += lam[i * 6 + j]; bi = fma(lam[i * 6 + j], li[j], bi); }
    b[i] = bi;
  }
}
// the prior log-likelihood li^T Lambda li
__device__ __forceinline__ double prior_quadratic(const double lam[36], const double li[6]) {
  double q = 0.0;
  for (int i = 0; i < 6; ++i) {
    double s = 0.0;
    for (int j = 0; j < 6; ++j) s = fma(lam[i * 6 + j], li[j], s);
    q = fma(li[i], s, q);
  }
  return q;
}

// The photometric mode's pose information: the Schur complement A_xx - A_xp A_pp^-1 A_px of the 8 x 8 system onto the pose,
// in fp64, with the 2 x 2 inverse written out.
__device__ __forceinline__ void schur_pose(const double A[64], double S[36]) {
  const double a = A[6 * 8 + 6], c = A[6 * 8 + 7], d = A[7 * 8 + 7];
  const double rdet = 1.0 / (a * d - c * c);
  const double i00 = d * rdet, i01 = -c * rdet, i11 = a * rdet;
  for (int i = 0; i < 6; ++i) {
    const double g0 = i00 * A[i * 8 + 6] + i01 * A[i * 8 + 7], g1 = i01 * A[i * 8 + 6] + i11 * A[i * 8 + 7];   // (A_pp^-1 A_px)^T row i
    for (int j = 0; j < 6; ++j) S[i * 6 + j] = A[i * 8 + j] - (g0 * A[j * 8 + 6] + g1 * A[j * 8 + 7]);
  }
}

// Smem: PairEndSmem, or PairEndSmemAffine for the photometric mode (8 unknowns: the 8 x 8 solve, the additive update of
// (alpha, beta), the Schur complement as the information, and the revert of (alpha, beta) with the pose).
template <typename Smem, typename Release>
__device__ __noinline__ void pair_end_cta(PairState& st, const PairLevel& pl, int pair, const double* partial, int ntiles,
                                             const LevelLaunch& lp, dvo_b200_iteration_stats* ilog, int max_log,
                                             Smem& sm, Release release, unsigned long long* tcrit = nullptr) {
  constexpr bool kAffine = Smem::kAffine;
  constexpr int kNV = kAffine ? kNormalValuesAffine : kNormalValues, kN = kAffine ? 8 : 6;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long tc0 = 0;
  if (tcrit && threadIdx.x == 0) asm volatile("mov.u64 %0, %globaltimer;" : "=l"(tc0));
  unsigned long long tph = tc0;
  // developer timing: ns per sub-phase of the end step into tcrit[k], the critical part into tcrit[7]
  auto phase = [&](int k) {
    if (tcrit) { unsigned long long tn; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(tn)); atomicAdd(tcrit + k, tn - tph); tph = tn; }
  };
  // fp64 sum of the level's strip partials in a fixed order: warp q takes strips q, q+4, ... with independent loads in flight;
  // lane l sums value l (and l + 32 in the photometric mode)
#pragma unroll
  for (int w0 = 0; w0 < kNV; w0 += 32) {
    double v = 0.0;
    if (w0 + lane < kNV && warp < kEndWarps) {
      const double* p = partial + (w0 + lane);
      int t = warp;
      for (; t + 3 * kEndWarps < ntiles; t += 4 * kEndWarps) {
        const double a0 = __ldcg(p + (size_t)t * kNV);
        const double a1 = __ldcg(p + (size_t)(t + kEndWarps) * kNV);
        const double a2 = __ldcg(p + (size_t)(t + 2 * kEndWarps) * kNV);
        const double a3 = __ldcg(p + (size_t)(t + 3 * kEndWarps) * kNV);
        v += a0; v += a1; v += a2; v += a3;
      }
      for (; t < ntiles; t += kEndWarps) v += __ldcg(p + (size_t)t * kNV);
    }
    if (warp < kEndWarps) sm.part[warp][w0 + lane] = v;
  }
  if constexpr (Smem::kPrior) {
    if (warp == kEndWarps) {
      const double* lam = sm.prior + (size_t)pair * 36;
      sm.lam[lane] = __ldg(lam + lane);
      if (lane < 4) sm.lam[32 + lane] = __ldg(lam + 32 + lane);
    }
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double vals[kNV];
#pragma unroll
  for (int i = 0; i < kNV; ++i) {
    double v = sm.part[0][i];
#pragma unroll
    for (int q = 1; q < kEndWarps; ++q) v += sm.part[q][i];
    vals[i] = v;
  }
  phase(0);   // partial sums

  // ---- critical ----
  const float P0 = st.precision[0], P1 = st.precision[1], P2 = st.precision[2], P3 = st.precision[3];
  // computeCompleteDataLogLikelihood: 0.5 n log det P - 3.5 sum log(1 + 0.2 d), returned as float
  const float det = __fsub_rn(__fmul_rn(P0, P3), __fmul_rn(P1, P2));
  const float logdet = (float)log((double)det);
  const float ll = (float)(0.5 * (double)st.n * (double)logdet - 0.5 * (5.0 + 2.0) * vals[0]);
  double li[6] = {0, 0, 0, 0, 0, 0};
  double sq = 0;
  if constexpr (Smem::kPrior) {
    se3_log(st.initial, li);                       // every pair: Lambda may be zero in some directions only
    sq = prior_quadratic(sm.lam, li);              // here, as sq by default: li need not live past the solve
  } else if (lp.mu != 0.0) {                       // mu == 0: prior term and the mu*log(initial) shift vanish
    se3_log(st.initial, li);
    for (int i = 0; i < 6; ++i) sq += li[i] * li[i];
  }
  phase(1);   // state loads, log, se3_log
  const double last_error = st.error;              // dense_tracking.cpp:306-307
  const double error = -(double)ll;
  const bool accept = error < last_error;          // dense_tracking.cpp:312
  double A[kN * kN], bvec[kN], x[kN];
  {
    int k = 1;
    for (int i = 0; i < kN; ++i)
      for (int j = i; j < kN; ++j) { A[i * kN + j] = vals[k]; A[j * kN + i] = vals[k]; ++k; }
    for (int i = 0; i < kN; ++i) bvec[i] = vals[1 + kN * (kN + 1) / 2 + i];
  }
  int iteration = st.iteration;
  const int it_id = iteration;                     // IterationStats.Id = itctx_.Iteration before the increment (dense_tracking.cpp:251)
  if (accept) {
    double As[kN * kN], bs[kN];
    for (int i = 0; i < kN * kN; ++i) As[i] = A[i];
    if constexpr (Smem::kPrior) {
      for (int i = 0; i < 6; ++i) bs[i] = bvec[i];
      add_prior<kN>(sm.lam, li, As, bs);
    } else {
      for (int i = 0; i < 6; ++i) { As[i * kN + i] += lp.mu; bs[i] = bvec[i] + lp.mu * li[i]; }   // lines 345-346 (the pose only)
    }
    if constexpr (kAffine) { bs[6] = bvec[6]; bs[7] = bvec[7]; }
    ldlt_solve<kN>(As, bs, x);                                                                   // line 347
    iteration += 1;                                                                              // line 353
  } else {
    for (int i = 0; i < 6; ++i) x[i] = st.x[i];
    if constexpr (kAffine) x[6] = x[7] = 0.0;
  }
  phase(2);   // accept test, LDL^T
  double m = 0; bool nanx = false;
  for (int i = 0; i < 6; ++i) { m = fmax(m, fabs(x[i])); nanx |= x[i] != x[i]; }
  const bool big = !nanx && m > lp.precision;
  const bool exceeded = iteration >= lp.max_iterations;
  const bool level_done = !(accept && big && !exceeded);                                       // line 357
  SE3d inc, estimate_new;
  if (!level_done) {
    // dense_tracking.cpp:259-263 for the next iteration: estimate = exp(x) * estimate, then K * float(T)
    inc = se3_exp(x);
    estimate_new = se3_mul(inc, st.estimate);
    double T[16];
    se3_matrix(estimate_new, T);
    // kt_of, open-coded: calling it here moves the photometric instances' spill slots
    for (int j = 0; j < 4; ++j) {
      const float t0 = (float)T[j], t1 = (float)T[4 + j], t2 = (float)T[8 + j];
      st.kt[j] = __fadd_rn(__fmul_rn(pl.cfx, t0), __fmul_rn(pl.cox, t2));
      st.kt[4 + j] = __fadd_rn(__fmul_rn(pl.cfy, t1), __fmul_rn(pl.coy, t2));
      st.kt[8 + j] = t2;
    }
    st.iteration = iteration;
    if constexpr (kAffine) {   // alpha += dalpha, beta += dbeta, with the pose
      AffineState& af = *sm.aff;
      const double a0 = af.ab[0], b0 = af.ab[1];
      af.ab_old[0] = a0; af.ab_old[1] = b0;
      af.ab[0] = a0 + x[6]; af.ab[1] = b0 + x[7];
    }
  } else {
    st.level_active = 0;
    if constexpr (kAffine) {   // a rejected iteration reverts (alpha, beta) with the pose
      AffineState& af = *sm.aff;
      if (!accept) { af.ab[0] = af.ab_old[0]; af.ab[1] = af.ab_old[1]; }
    }
  }
  phase(3);   // exp, pose product, K*T
  if (tcrit) { unsigned long long tc1; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(tc1)); atomicAdd(tcrit + 7, tc1 - tc0); }
  release();
  phase(4);   // release

  // ---- deferred ----
  LevelSummary& ls = st.levels[lp.level_index];
  st.ll = ll;
  st.nll_cur = -(double)ll;
  if constexpr (Smem::kPrior) st.prior_cur = sq;   // li^T Lambda li
  else st.prior_cur = lp.mu * sq;                  // dense_tracking.cpp:302
  st.last_error = last_error;
  st.error = error;
  if constexpr (kAffine) {
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j < 6; ++j) st.A[i * 6 + j] = A[i * kN + j];
  } else {
    for (int i = 0; i < 36; ++i) st.A[i] = A[i];
  }
  for (int i = 0; i < 6; ++i) st.b[i] = bvec[i];
  if constexpr (kAffine) {
    if (sm.keep_system) {
      for (int i = 0; i < 64; ++i) sm.aff->A[i] = A[i];
      for (int i = 0; i < 8; ++i) sm.aff->b[i] = bvec[i];
    }
  }
  if (!accept) {
    st.initial = st.initial_old; st.estimate = st.estimate_old;   // dense_tracking.cpp:314-321
    st.termination = DVO_B200_TERM_LOG_LIKELIHOOD_DECREASED;
    log_iteration(ilog, max_log, pair, st, it_id, lp.level_id, false);
  } else {
    for (int i = 0; i < 6; ++i) st.x[i] = x[i];
    if constexpr (kAffine) {
      double Ap[64];
      for (int i = 0; i < 64; ++i) Ap[i] = A[i];
      if constexpr (Smem::kPrior) {
        for (int i = 0; i < 6; ++i)
          for (int j = 0; j < 6; ++j) Ap[i * 8 + j] += sm.lam[i * 6 + j];
      } else {
        for (int i = 0; i < 6; ++i) Ap[i * 8 + i] += lp.mu;
      }
      schur_pose(Ap, st.A_done);
    } else {
      for (int i = 0; i < 36; ++i) st.A_done[i] = A[i];
      if constexpr (Smem::kPrior) {
        for (int i = 0; i < 36; ++i) st.A_done[i] += sm.lam[i];
      } else {
        for (int i = 0; i < 6; ++i) st.A_done[i * 6 + i] += lp.mu;
      }
    }
    st.nll_done = st.nll_cur; st.prior_done = st.prior_cur; st.have_done = 1;
    ls.last_inc_n = st.n; ls.last_inc_nll = st.nll_cur;
    log_iteration(ilog, max_log, pair, st, it_id, lp.level_id, true);
    st.iteration = iteration;
  }
  if (level_done) {
    if (!nanx && m <= lp.precision) st.termination = DVO_B200_TERM_INCREMENT_TOO_SMALL;       // line 359
    if (exceeded) st.termination = DVO_B200_TERM_ITERATIONS_EXCEEDED;                         // line 362
    ls.termination = st.termination;
    int need = (st.termination == DVO_B200_TERM_LOG_LIKELIHOOD_DECREASED ||
                st.termination == DVO_B200_TERM_TOO_FEW_CONSTRAINTS) ? 2 : 1;
    ls.has_inc = ls.num_iterations >= need;
  } else {
    st.inc = inc;
    st.initial_old = st.initial;
    st.initial = se3_mul(se3_inverse(inc), st.initial);
    st.estimate_old = st.estimate;
    st.estimate = estimate_new;
  }
  phase(5);   // deferred bookkeeping
}

// ------------------------------------------------------------------------------------------------
// The persistent cooperative level kernel.
//
// The grid is num_sms x C CTAs (C = resident CTAs per SM, 2 with 95-97 KB of shared memory each) of 8 warps.  CTAs are
// grouped into squads of g CTAs; a squad owns ONE frame pair at a time, CTA r of the squad the strips r, r+g, r+2g, ...
// (kTileH image rows each), and runs all its Gauss-Newton iterations on the segment's levels inside the kernel:
//   stage A over the CTA's tiles -> per-row scale summaries -> per-strip summaries (fp64) -> squad barrier, the last
//   CTA to arrive combines the level's strips and computes P_k (pair_mid_warp) -> stage B -> per-row sums -> per-strip
//   sums (fp64) -> squad barrier, the last CTA adds the level's strips, tests the log-likelihood, solves the 6x6
//   system and updates the pose (pair_end_cta) -> next iteration,
// then takes the next pair from a global queue.  The two resident CTAs of an SM belong to different squads, so
// one squad's barrier wait is hidden by the other.
// ------------------------------------------------------------------------------------------------
struct SquadState {
  int pair;
  unsigned arrive;
  unsigned phase;
  int pad_[29];   // one 128-byte line per squad
};

template <bool kAffine, bool kPrior = false>
struct LevelTailOf {    // shared memory after the tile pipeline
  using EndBase = typename std::conditional<kAffine, PairEndSmemAffine, PairEndSmem>::type;
  SegCombineSmem comb;
  typename std::conditional<kPrior, PairEndSmemPrior<EndBase>, EndBase>::type end;
  int s_flag[2];
};
template <bool kAffine, bool kPrior = false>
constexpr size_t kLevelSmemBytesOf = sizeof(TilePipe) + sizeof(LevelTailOf<kAffine, kPrior>);
// Two resident CTAs per SM: an H100 SM has up to 228 KB of shared memory and reserves 1 KB of it per resident CTA.  (With
// the default window, kWinRows of stages.cuh, two CTAs take at most 196 KB, the carveout that leaves 60 KB of L1.)
constexpr size_t kSmemPerSm = 228 * 1024, kSmemReservedPerCta = 1024;

// One segment of a launch: a group of consecutive pyramid levels that a squad of g CTAs walks a pair through.  A launch
// has one segment, or two (the coarse levels with one CTA per pair, then the fine levels with squads of g CTAs) that the
// grid runs back to back WITHOUT a grid-wide barrier: a CTA that finds the coarse queue empty moves on to the fine
// segment, and fine squads take their pairs from a ring of pairs whose coarse levels are done (`ready`).
struct Segment {
  const PairLevel* pls;   // descriptors of this segment's levels: [level][pair]
  float* row_exports;     // per squad: h segment summaries (one per image row)
  int* row_base;          // per squad: h exclusive prefixes of valid counts, relative to the owning CTA's first row
  double* strip_exports;  // per squad: one scale summary per strip (kStripExportDoubles)
  int* strip_base;        // per squad: nstrips + 1 exclusive prefixes of the strips' valid counts
  float* row_partial;     // per squad: kNormalValues per image row (stage B)
  double* strip_partial;  // per squad: kNormalValues per strip, the strip's rows summed in fp64
  SquadState* squads;
  int* queue;             // next pair (first segment) / next slot of this segment's ready ring (later segments of a fused launch)
  int* ready;             // fused launch, segments >= 1: ring of (pair + 1) whose coarse levels are done, 0 = not yet written
  int* ready_tail;
  int* arrivals;          // CTAs that have entered this segment (squads of segments >= 1 form in order of arrival)
  int cyclic;             // 1: CTA r of a squad takes strips r, r + g, ...; 0: contiguous ranges of strips_per_cta strips
  int pair_begin;         // segments >= 1 of a fused launch own the pairs [pair_begin, pair_begin + npairs_seg)
  int npairs_seg;         // pairs handed out by this segment's queue
  unsigned long long* dbg2;  // optional (timing build): {tiles, inexact tiles, skipped tiles, rounds, stage-B rounds in the generic loop, max / min CTA lifetime}
  unsigned long long* dbg;   // optional: ns spent per CTA in {stage A, stage B, wait A, wait B, mid, end, queue, total}
  int nlev;               // pyramid levels of the segment (coarse to fine)
  int g, nsquads;
  int strips_per_cta[kMaxLevels];
  LevelLaunch lp[kMaxLevels];
};

struct PersistentArgs {
  PairState* states;
  int* error_flag;
  dvo_b200_iteration_stats* ilog;
  int max_log;
  const double* T_init;   // per pair 4x4 (device memory) or nullptr
  int skip_begin;         // test hook: the pair state was placed by k_set_state
  float* dump;            // test hook: seven record planes of the (single) pair, or nullptr
  int npairs;
  int nseg;               // 1, or >= 2 = fused launch: coarse segment + slices of the fine levels
  Segment seg[kMaxSeg];
  const PairLevel* pls0;  // kCurMask: csat[i] belongs to the descriptor pls0[i]
  const int* const* csat;
  AffineState* affine;    // kAffine: per pair
  const double* prior;    // kPrior: per pair the 6 x 6 prior information Lambda, row-major (device memory)
};

// The descriptor of one pair at one level of a segment: a PairLevel, or with kCurMask a CurPairLevel.
template <bool kCurMask> struct LevelOf {
  using type = PairLevel;
  static __device__ __forceinline__ PairLevel load(const PersistentArgs& a, const Segment& S, size_t i) { return S.pls[i]; }
};
template <> struct LevelOf<true> {
  using type = CurPairLevel;
  static __device__ __forceinline__ CurPairLevel load(const PersistentArgs& a, const Segment& S, size_t i) {
    CurPairLevel q;
    static_cast<PairLevel&>(q) = S.pls[i];
    q.csat = a.csat[(size_t)(S.pls - a.pls0) + i];
    return q;
  }
};

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// returns true in every thread of the CTA that arrived last at barrier episode `episode`
__device__ __forceinline__ bool squad_arrive(SquadState* sq, unsigned episode, int g, int* s_flag) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    unsigned old = atomicAdd(&sq->arrive, 1u);
    int last = old == (episode + 1u) * (unsigned)g - 1u;
    if (last) __threadfence();
    s_flag[0] = last;
  }
  __syncthreads();
  return s_flag[0] != 0;
}
__device__ __forceinline__ void squad_release(SquadState* sq, unsigned episode) {
  __threadfence();
  atomicExch(&sq->phase, episode + 1u);
}
__device__ __forceinline__ void squad_wait(SquadState* sq, unsigned episode, int* error_flag) {
  if (threadIdx.x == 0) {
    unsigned spins = 0;
    while (ld_acquire_u32(&sq->phase) < episode + 1u) {
      __nanosleep(100);
      if (((++spins) & 4095u) == 0u) {
        if (*reinterpret_cast<volatile int*>(error_flag)) break;
        if (spins > (1u << 25)) { atomicExch(error_flag, 1); break; }   // ~ seconds: never hang the GPU
      }
    }
  }
  __syncthreads();
}

// kCorrected: the corrected estimator (dvo_b200_estimator), one instance per value, chosen per launch.
// kCurMask: some pair's current image has a mask in the current role (PairLevel::csat); stage B then tests the taps of the
// tiles whose window touches an unusable pixel (produce_tiles, stage_b_rounds).  Without it the instance is the one that
// existed before current-role masks.
// kAffine: the photometric mode (include/dvo_b200.h): a gain and a bias per pair (PersistentArgs::affine) estimated with the
// pose, 45 normal-equation values per row instead of 28.  Its stage-B loop holds 17 more accumulators; it is compiled for
// kAffineCtasPerSm resident CTAs (DESIGN §4.8), and the launch plan of a photometric match uses that occupancy.
#ifndef DVO_AFFINE_CTAS_PER_SM
#define DVO_AFFINE_CTAS_PER_SM 2
#endif
constexpr int kAffineCtasPerSm = DVO_AFFINE_CTAS_PER_SM;
// kPrior: a 6 x 6 prior information per pair (PersistentArgs::prior) in place of mu I in the end step (include/dvo_b200.h,
// "motion prior"); the pixel loops are those of the instance without it.
template <bool kCorrected, bool kCurMask = false, bool kAffine = false, bool kPrior = false>
__global__ void __launch_bounds__(kCtaThreads, kAffine ? kAffineCtasPerSm : 2)
k_level_persistent(const __grid_constant__ PersistentArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  TilePipe& tp = *reinterpret_cast<TilePipe*>(smem_raw);
  LevelTailOf<kAffine, kPrior>& lt = *reinterpret_cast<LevelTailOf<kAffine, kPrior>*>(smem_raw + sizeof(TilePipe));
  constexpr int kNV = kAffine ? kNormalValuesAffine : kNormalValues;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&tp.full[i], 1); mbar_init(&tp.empty[i], kConsumerWarps); }
    mbar_fence_init();
    if constexpr (kPrior) lt.end.prior = a.prior;
  }
  __syncthreads();
  unsigned tile_count = 0;      // tiles staged / consumed by this CTA since the kernel started
  const bool fused = a.nseg >= 2;
#define DVO_TICK() do { if (timing) t0 = global_ns(); } while (0)
#define DVO_TOCK(slot) do { if (timing) { t1 = global_ns(); t_acc[slot] += t1 - t0; t0 = t1; } } while (0)

#pragma unroll 1
  for (int si = 0; si < a.nseg; ++si) {
  const Segment& S = a.seg[si];
  // Squads of the second segment of a fused launch form in ORDER OF ARRIVAL: the CTAs leave the first segment at very
  // different times (1 or 2 coarse pairs each, 3..40 iterations per level), and a squad made of neighbouring block indices
  // would wait for its slowest member.
  int cta_index = blockIdx.x;
  if (fused && si >= 1) {
    if (threadIdx.x == 0) lt.s_flag[1] = atomicAdd(S.arrivals, 1);
    __syncthreads();
    cta_index = lt.s_flag[1];
    __syncthreads();
  }
  const int squad = cta_index / S.g, rank = cta_index - squad * S.g;
  if (squad >= S.nsquads) continue;   // leftover CTAs of this segment
  SquadState* sq = S.squads + squad;
  int hmax = 0;
  for (int li = 0; li < S.nlev; ++li) hmax = max(hmax, S.lp[li].h);
  float* row_exports = S.row_exports + (size_t)squad * hmax * kSegExportFloats;
  int* row_base = S.row_base + (size_t)squad * hmax;
  const int smax = (hmax + kTileH - 1) / kTileH;      // strips of the tallest level of the segment
  double* strip_exports = S.strip_exports + (size_t)squad * smax * kStripExportDoubles;
  int* strip_base = S.strip_base + (size_t)squad * (smax + 1);
  float* row_partial = S.row_partial + (size_t)squad * hmax * kNV;
  double* strip_partial = S.strip_partial + (size_t)squad * smax * kNV;
  unsigned episode = 0;
  unsigned long long t_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, t0 = 0, t1 = 0;
  const bool timing = S.dbg != nullptr && threadIdx.x == 0;
  PipeTiming tm;
#ifdef DVO_PIPE_TIMING
  tm.on = S.dbg != nullptr && lane == 0 && (warp == 0 || warp == kConsumerWarps);   // one consumer warp and the producer
#endif
  const unsigned long long t_start = timing ? global_ns() : 0;

  for (;;) {
    DVO_TICK();
    // ---- take the next pair from the queue (the last CTA to arrive does it for the squad) ----
    if (squad_arrive(sq, episode, S.g, lt.s_flag)) {
      if (threadIdx.x == 0) {
        int p = atomicAdd(S.queue, 1);
        if (p >= S.npairs_seg) p = -1;
        else if (fused && si >= 1) {
          // slot p of this segment's ready ring: filled by the CTA that finishes the coarse levels of one of the
          // segment's pairs (every pair is pushed exactly once, so every slot < npairs_seg is eventually written)
          unsigned spins = 0;
          int v;
          while ((v = (int)ld_acquire_u32(reinterpret_cast<const unsigned*>(S.ready + p))) == 0) {
            __nanosleep(200);
            if (((++spins) & 4095u) == 0u) {
              if (*reinterpret_cast<volatile int*>(a.error_flag)) break;
              if (spins > (1u << 24)) { atomicExch(a.error_flag, 1); break; }
            }
          }
          p = v - 1;
        }
        sq->pair = p;
        squad_release(sq, episode);
      }
    } else {
      squad_wait(sq, episode, a.error_flag);
    }
    __syncthreads();
    ++episode;
    DVO_TOCK(6);
    const int pair = __ldcg(&sq->pair);
    if (pair < 0 || *reinterpret_cast<volatile int*>(a.error_flag)) break;
    PairState& st = a.states[pair];
    // (alpha, beta) of the pair's current iteration, read like the pose (written between stages by another SM)
    auto brightness = [&]() {
      Brightness br{1.f, 0.f};
      if constexpr (kAffine) br = Brightness{(float)__ldcg(&a.affine[pair].ab[0]), (float)__ldcg(&a.affine[pair].ab[1])};
      return br;
    };

    // ---- the squad walks its pair through the levels of this launch, coarse to fine ----
    for (int li = 0; li < S.nlev; ++li) {
    const LevelLaunch& lp = S.lp[li];
    const typename LevelOf<kCurMask>::type pl = LevelOf<kCurMask>::load(a, S, (size_t)li * a.npairs + pair);
    LevelGeom geo;
    geo.w = lp.w; geo.h = lp.h; geo.n = lp.n; geo.pitch = lp.pitch; geo.nbands = lp.nbands; geo.nstrips = lp.nstrips;
    if (S.cyclic) {   // CTA r takes strips r, r + g, r + 2g, ...: every CTA of the squad samples the whole image
      const int g_eff = min(S.g, lp.nstrips);
      geo.strip0 = min(rank, lp.nstrips); geo.strip_step = g_eff;
      geo.nmine = rank < g_eff ? (lp.nstrips - rank + g_eff - 1) / g_eff : 0;
    } else {          // contiguous ranges
      geo.strip0 = min(rank * S.strips_per_cta[li], lp.nstrips); geo.strip_step = 1;
      geo.nmine = min(geo.strip0 + S.strips_per_cta[li], lp.nstrips) - geo.strip0;
    }
    if (!a.skip_begin) {   // DenseTracker::match, start of a level: the last CTA to arrive initialises the pair's level state
      if (squad_arrive(sq, episode, S.g, lt.s_flag)) {
        if (threadIdx.x == 0) {
          level_begin(st, pl, a.T_init, pair, lp);
          if constexpr (kAffine) {   // the level's first iteration reverts (alpha, beta) to where the level starts
            AffineState& af = a.affine[pair];
            af.ab_old[0] = af.ab[0]; af.ab_old[1] = af.ab[1];
          }
          squad_release(sq, episode);
        }
      } else {
        squad_wait(sq, episode, a.error_flag);
      }
      __syncthreads();
      ++episode;
      DVO_TOCK(6);
    }

    for (;;) {
      // ---- stage A ----
      {
        StageConsts c;
        load_stage_consts(st, pl, lp.w, lp.h, false, c);
        const long long ts0 = DVO_CLOCK(tm);
        stage_a_run<kCorrected, kAffine>(tp, pl, geo, c, row_exports, tile_count, a.error_flag, tm, brightness());
        DVO_ADD(tm, rounds_a, DVO_CLOCK(tm) - ts0);
      }
      __syncthreads();
      // this CTA's strips: the rows of a strip in order -> the strip's summary (one thread per strip); row_base: rank of each
      // row's first point inside its strip
      for (int j = threadIdx.x; j < geo.nmine; j += kCtaThreads) {
        const int sj = geo.strip0 + j * geo.strip_step;
        combine_strip_rows(row_exports, sj * kTileH, min(sj * kTileH + kTileH, lp.h), row_base, strip_exports + (size_t)sj * kStripExportDoubles);
      }
      DVO_TOCK(0);
      if (squad_arrive(sq, episode, S.g, lt.s_flag)) {
        DVO_TOCK(2);
        if (warp == 0) {
          pair_mid_warp<kCorrected>(st, pair, strip_exports, strip_base, lp.nstrips, lp, a.ilog, a.max_log, lt.comb);
          if constexpr (kAffine) {   // too few constraints: the pose was reverted, and (alpha, beta) go with it
            AffineState& af = a.affine[pair];
            if (lane == 0 && !st.level_active) {   // and, as the pose's, no normal equations for the linearisation hook
              af.ab[0] = af.ab_old[0]; af.ab[1] = af.ab_old[1];
              if (a.skip_begin) {
                for (int i = 0; i < 64; ++i) af.A[i] = 0.0;
                for (int i = 0; i < 8; ++i) af.b[i] = 0.0;
              }
            }
          }
          if (lane == 0) squad_release(sq, episode);
        }
        __syncthreads();
        DVO_TOCK(4);
      } else {
        squad_wait(sq, episode, a.error_flag);
        DVO_TOCK(2);
      }
      __syncthreads();
      ++episode;
      // too few constraints: the level ends here.  The residual-image hook still gets this iteration's records, so with a
      // dump the CTA runs stage B once more for the dump alone (its sums are discarded).
      const bool failed = *reinterpret_cast<volatile int*>(a.error_flag) != 0;
      const bool level_ends = failed || !__ldcg(&st.level_active);
      if (level_ends && (!a.dump || failed)) break;

      // ---- stage B ----
      {
        StageConsts c;
        load_stage_consts(st, pl, lp.w, lp.h, true, c);
        StageBConsts cb;
        load_stage_b_consts(st, cb);
        const long long n_keep = __ldcg(&st.n_keep);
        RecordDump dump;
        dump.planes = a.dump; dump.n = lp.n;
        const long long ts0 = DVO_CLOCK(tm);
        const Brightness br = brightness();
        if (a.dump) stage_b_run<true, kCorrected, kCurMask, kAffine>(tp, pl, geo, c, cb, row_base, strip_base, n_keep, dump, row_partial, tile_count, a.error_flag, tm, br);
        else stage_b_run<false, kCorrected, kCurMask, kAffine>(tp, pl, geo, c, cb, row_base, strip_base, n_keep, dump, row_partial, tile_count, a.error_flag, tm, br);
        DVO_ADD(tm, rounds_b, DVO_CLOCK(tm) - ts0);
      }
      __syncthreads();
      if (level_ends) break;
      // the rows of each of this CTA's strips, in order, in fp64: one thread per (strip, value)
      for (int it = threadIdx.x; it < geo.nmine * kNV; it += kCtaThreads) {
        const int j = it / kNV, i = it - j * kNV;
        const int sj = geo.strip0 + j * geo.strip_step;
        const int nrow = min(kTileH, lp.h - sj * kTileH);
        const float* rp = row_partial + (size_t)sj * kTileH * kNV + i;
        float r[kTileH];
#pragma unroll
        for (int k = 0; k < kTileH; ++k) r[k] = k < nrow ? __ldcg(rp + (size_t)k * kNV) : 0.f;   // independent loads
        double v = 0.0;
#pragma unroll
        for (int k = 0; k < kTileH; ++k) v += (double)r[k];      // a missing row adds an exact zero
        strip_partial[(size_t)sj * kNV + i] = v;
      }
      DVO_TOCK(1);
      if (squad_arrive(sq, episode, S.g, lt.s_flag)) {
        DVO_TOCK(3);
        if constexpr (kAffine) {
          if (threadIdx.x == 0) { lt.end.aff = a.affine + pair; lt.end.keep_system = a.skip_begin; }
        }
        pair_end_cta(st, pl, pair, strip_partial, lp.nstrips, lp, a.ilog, a.max_log, lt.end, [&] { squad_release(sq, episode); }, S.dbg2 ? S.dbg2 + 64 : nullptr);
        __syncthreads();
        DVO_TOCK(5);
      } else {
        squad_wait(sq, episode, a.error_flag);
        DVO_TOCK(3);
      }
      __syncthreads();
      ++episode;
      if (!__ldcg(&st.level_active) || *reinterpret_cast<volatile int*>(a.error_flag)) break;
    }
    if (*reinterpret_cast<volatile int*>(a.error_flag)) break;
    }   // levels
    if (fused && si == 0 && threadIdx.x == 0) {   // this pair's coarse levels are done: hand it to the fine squads (g == 1 here)
      // The fine segments own fixed ranges of the pair index (not of the order of arrival), so which squad size a pair
      // gets -- and with it the rounding of its sums -- does not depend on timing.
      int k = 1;
      while (k + 1 < a.nseg && pair >= a.seg[k + 1].pair_begin) ++k;
      __threadfence();
      const int slot = atomicAdd(a.seg[k].ready_tail, 1);
      asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(a.seg[k].ready + slot), "r"(pair + 1) : "memory");
    }
  }
  if (timing) {
    t_acc[7] = global_ns() - t_start;
    for (int i = 0; i < 8; ++i) atomicAdd(S.dbg + i, t_acc[i]);
  }
#ifdef DVO_PIPE_TIMING
  if (tm.on) {   // cycles: consumer warp 0 {stage A, wait full A, stage B, wait full B}, producer {descriptor, wait empty}
    if (warp == 0) { atomicAdd(S.dbg + 8, tm.rounds_a); atomicAdd(S.dbg + 9, tm.wait_full_a); atomicAdd(S.dbg + 10, tm.rounds_b); atomicAdd(S.dbg + 11, tm.wait_full_b); }
    else { atomicAdd(S.dbg + 12, tm.produce); atomicAdd(S.dbg + 13, tm.wait_empty); atomicAdd(S.dbg + 14, tm.rounds_a); atomicAdd(S.dbg + 15, tm.rounds_b); }
    if (warp == 0) { atomicAdd(S.dbg2 + 3, tm.rounds); atomicAdd(S.dbg2 + 4, tm.slow_rounds); }
    else { atomicAdd(S.dbg2 + 0, tm.tiles); atomicAdd(S.dbg2 + 1, tm.tiles_inexact); atomicAdd(S.dbg2 + 2, tm.tiles_skipped); atomicAdd(S.dbg2 + 7, tm.tiles_cmask); }
  }
  if (timing) { atomicMax(S.dbg2 + 5, t_acc[7]); atomicMin(S.dbg2 + 6, t_acc[7]); }
#endif
  }   // segments
#undef DVO_TICK
#undef DVO_TOCK
}

// Result assembly (dense_tracking.cpp:368-373)
__global__ void k_finalize(PairState* states, dvo_b200_result* results, int npairs) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= npairs) return;
  PairState& st = states[p];
  dvo_b200_result& r = results[p];
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  se3_matrix(se3_inverse(st.estimate), r.transformation);
  // last_iteration = Iterations[size-1] unless LogLikelihoodDecreased (then size-2).  With
  // TooFewConstraints on the last level, or no completed iteration, the reference reads an
  // uninitialised / out-of-range element (SURVEY Q24); defined here as NaN so Result::isNaN() fires.
  bool ok = st.result_defined();
  for (int i = 0; i < 36; ++i) r.information[i] = ok ? st.A_done[i] * 0.008 * 0.008 : nan;
  r.log_likelihood = ok ? st.nll_done + st.prior_done : nan;
  r.num_levels = st.num_levels;
  r.num_iterations_total = st.num_iterations_total;
  for (int l = 0; l < kMaxLevels; ++l) {
    dvo_b200_level_stats& o = r.levels[l];
    if (l < st.num_levels) {
      const LevelSummary& s = st.levels[l];
      o.id = s.id; o.termination = s.termination; o.max_valid_pixels = s.max_valid_pixels;
      o.valid_pixels = s.valid_pixels; o.num_iterations = s.num_iterations;
      o.has_iteration_with_increment = s.has_inc; o.last_valid_constraints = s.last_n;
      o.last_increment_valid_constraints = s.last_inc_n; o.last_increment_log_likelihood = s.last_inc_nll;
    } else {
      o.id = -1; o.termination = -1; o.max_valid_pixels = 0; o.valid_pixels = 0; o.num_iterations = 0;
      o.has_iteration_with_increment = 0; o.last_valid_constraints = 0; o.last_increment_valid_constraints = -1;
      o.last_increment_log_likelihood = nan;
    }
  }
}

// test hook: place a fixed transform / precision / iteration flag into the state (no exp/log chain)
// (prev_precision: the precision of the previous iteration, 0 without weights)
__global__ void k_set_state(PairState* states, const PairLevel* pls, const double* T, float4 prev_precision, int use_weights,
                            LevelLaunch lp) {
  PairState& st = states[0];
  const PairLevel& pl = pls[0];
  st.estimate = se3_from_matrix(T); st.estimate_old = st.estimate;
  st.initial = se3_identity(); st.initial_old = st.initial; st.inc = se3_identity();
  for (int i = 0; i < 6; ++i) st.x[i] = 0;
  st.iteration = use_weights ? 1 : 0;
  st.precision[0] = prev_precision.x; st.precision[1] = prev_precision.y; st.precision[2] = prev_precision.z;
  st.precision[3] = prev_precision.w;
  st.error = 1.7976931348623157e308; st.last_error = st.error;
  st.level_active = 1; st.phase_ok = 0; st.have_done = 0; st.termination = -1;
  st.num_levels = 1; st.num_iterations_total = 0; st.iter_log_count = 0;
  LevelSummary& ls = st.levels[0];
  ls.id = lp.level_id; ls.num_iterations = 0; ls.valid_pixels = pl.rsel[0]; ls.max_valid_pixels = pl.max_valid_pixels;
  // take the matrix exactly as given (the round trip through the quaternion is not bit exact)
  kt_of(T, pl, st.kt);
}

// (alpha, beta) of the photometric mode at the start of a match or test hook: ab (2n doubles, pinned host memory read over
// PCIe, or NULL = (1, 0) each)
__global__ void k_affine_init(AffineState* s, const double* ab, int n) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  const double a = ab ? ab[2 * p] : 1.0, b = ab ? ab[2 * p + 1] : 0.0;
  s[p].ab[0] = a; s[p].ab[1] = b; s[p].ab_old[0] = a; s[p].ab_old[1] = b;
}

// Multi-hypothesis alignment, between the screening and the continuation: one warp per pair p.  The scores of its k screened
// hypotheses (states p k .. p k + k - 1, their statistics of the screening level at level index ls) go to scores[p k + j]
// (hypothesis_score), the choice to best[p] (pick_hypothesis), and the chosen hypothesis's state and first
// min(iter_log_count, max_log) iteration-log entries to slot p of the continuation, which picks up from there.  kAffine: the
// chosen hypothesis's AffineState follows its state (screened_aff -> chosen_aff); kPrior: its 36 doubles of Lambda
// (screened_prior -> chosen_prior).  The <false, false> instance ignores those four arguments.
template <bool kAffine, bool kPrior>
__global__ void k_pick_hypotheses(const PairState* __restrict__ screened, const dvo_b200_iteration_stats* __restrict__ screened_log,
                                  PairState* __restrict__ chosen, dvo_b200_iteration_stats* __restrict__ chosen_log, int max_log, int n,
                                  int k, int ls, double min_ratio, double* __restrict__ scores, int* __restrict__ best,
                                  const AffineState* __restrict__ screened_aff, AffineState* __restrict__ chosen_aff,
                                  const double* __restrict__ screened_prior, double* __restrict__ chosen_prior) {
  const int p = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (p >= n) return;
  double* const sc = scores + (size_t)p * k;
  for (int j = lane; j < k; j += 32) {
    const LevelSummary& L = screened[(size_t)p * k + j].levels[ls];
    sc[j] = hypothesis_score(L.has_inc, L.last_inc_n, L.valid_pixels, L.last_inc_nll, min_ratio);
  }
  __syncwarp();
  int b = 0;
  if (lane == 0) {
    b = pick_hypothesis(sc, k);
    best[p] = b;
  }
  b = __shfl_sync(kFull, b, 0);
  static_assert(sizeof(PairState) % 8 == 0 && sizeof(dvo_b200_iteration_stats) % 8 == 0, "copied as 8-byte words");
  const PairState& src = screened[(size_t)p * k + b];
  const unsigned long long* s = reinterpret_cast<const unsigned long long*>(&src);
  unsigned long long* d = reinterpret_cast<unsigned long long*>(chosen + p);
  for (int i = lane; i < (int)(sizeof(PairState) / 8); i += 32) d[i] = s[i];
  if (max_log > 0) {
    const size_t words = (size_t)min(src.iter_log_count, max_log) * (sizeof(dvo_b200_iteration_stats) / 8);
    const unsigned long long* ls8 = reinterpret_cast<const unsigned long long*>(screened_log + ((size_t)p * k + b) * max_log);
    unsigned long long* ld8 = reinterpret_cast<unsigned long long*>(chosen_log + (size_t)p * max_log);
    for (size_t i = lane; i < words; i += 32) ld8[i] = ls8[i];
  }
  if constexpr (kAffine) {
    static_assert(sizeof(AffineState) % 8 == 0, "copied as 8-byte words");
    const unsigned long long* a = reinterpret_cast<const unsigned long long*>(screened_aff + (size_t)p * k + b);
    unsigned long long* ad = reinterpret_cast<unsigned long long*>(chosen_aff + p);
    for (int i = lane; i < (int)(sizeof(AffineState) / 8); i += 32) ad[i] = a[i];
  }
  if constexpr (kPrior) {
    const double* lam = screened_prior + ((size_t)p * k + b) * 36;
    for (int i = lane; i < 36; i += 32) chosen_prior[(size_t)p * 36 + i] = lam[i];
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// The k_level_persistent instance of a call: its template flags, decided once per call.
struct LevelVariant {
  bool corrected;   // ctx->estimator is the corrected estimator
  bool cur_mask;    // some pair's current pyramid has a mask in the current role (any_current_mask)
  bool affine;      // the photometric mode
  bool prior;       // a motion prior per pair
};

struct LevelInstance {
  const void* kernel;
  size_t smem;      // dynamic shared memory
};
template <bool kAffine, bool kPrior>
LevelInstance level_instance_of(const LevelVariant& v) {
  static_assert(2 * (kLevelSmemBytesOf<kAffine, kPrior> + kSmemReservedPerCta) <= kSmemPerSm, "two CTAs of the level kernel must fit on an SM");
  const void* const k[2][2] = {
      {(const void*)k_level_persistent<false, false, kAffine, kPrior>, (const void*)k_level_persistent<false, true, kAffine, kPrior>},
      {(const void*)k_level_persistent<true, false, kAffine, kPrior>, (const void*)k_level_persistent<true, true, kAffine, kPrior>}};
  return {k[v.corrected][v.cur_mask], kLevelSmemBytesOf<kAffine, kPrior>};
}
LevelInstance level_instance(const LevelVariant& v) {
  if (v.prior) return v.affine ? level_instance_of<true, true>(v) : level_instance_of<false, true>(v);
  return v.affine ? level_instance_of<true, false>(v) : level_instance_of<false, false>(v);
}

// The grid of v's instances: the smallest occupancy of the four (estimator x current mask) that share v's photometric mode
// and prior.  Each such group is set up on its first use, so that the default grid comes from the default instances alone.
int ensure_geometry(dvo_b200_ctx* ctx, const LevelVariant& v) {
  int& cached = ctx->ctas_per_sm[v.affine][v.prior];
  if (cached != 0) return 0;
  if (ctx->num_sms == 0) DVO_CUDA(ctx, cudaDeviceGetAttribute(&ctx->num_sms, cudaDevAttrMultiProcessorCount, ctx->device));
  int per_sm = 1 << 30;
  for (int k = 0; k < 4; ++k) {
    const LevelInstance li = level_instance({(k & 1) != 0, (k & 2) != 0, v.affine, v.prior});
    DVO_CUDA(ctx, cudaFuncSetAttribute(li.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)li.smem));
    int k_per_sm = 0;
    DVO_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&k_per_sm, li.kernel, kCtaThreads, li.smem));
    per_sm = std::min(per_sm, k_per_sm);
  }
  if (per_sm < 1)
    return set_error(ctx, DVO_B200_ERR_CUDA, std::string("persistent kernel") + (v.prior ? " (motion prior)" : v.affine ? " (photometric)" : "")
                                                 + " does not fit on an SM");
  cached = per_sm;
  return 0;
}

int grid_ctas(const dvo_b200_ctx* ctx, const LevelVariant& v) { return ctx->num_sms * ctx->ctas_per_sm[v.affine][v.prior]; }

// Byte offsets of one launch's scratch in the workspace arena, every region on a 128-byte boundary.  Per segment, for each
// of its squads and sized for the segment's tallest level: the row and strip scale summaries, the valid-count prefixes of
// rows and strips, and the row and strip partials of the normal equations.  Then the squad states of every segment, the
// counter line and the ready ring, back to back so that one memset zeroes them before the launch.
struct ScratchLayout {
  size_t row_exports[kMaxSeg], row_base[kMaxSeg], strip_exports[kMaxSeg], strip_base[kMaxSeg], row_partial[kMaxSeg],
         strip_partial[kMaxSeg], squads[kMaxSeg];
  size_t counters;   // one 128-byte line: {queue[kMaxSeg], ready tail[kMaxSeg], arrivals[kMaxSeg], error flag}
  size_t ring;       // npairs slots: the ready rings of the fine segments, by pair range
  size_t bytes;
};

// nvals: normal-equation values per row and strip (kNormalValues, or kNormalValuesAffine in the photometric mode)
ScratchLayout scratch_layout(const PlanLaunch& L, int npairs, int nvals) {
  ScratchLayout o;
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t off = at; at += (bytes + 127) / 128 * 128; return off; };
  for (int s = 0; s < L.nseg; ++s) {
    const PlanSegment& S = L.seg[s];
    const size_t rows = (size_t)S.nsquads * S.hmax, strips = (size_t)S.nsquads * ((S.hmax + kTileH - 1) / kTileH);
    o.row_exports[s] = take(sizeof(float) * kSegExportFloats * rows);
    o.row_base[s] = take(sizeof(int) * rows);
    o.strip_exports[s] = take(sizeof(double) * kStripExportDoubles * strips);
    o.strip_base[s] = take(sizeof(int) * (strips + S.nsquads));   // nstrips + 1 per squad
    o.row_partial[s] = take(sizeof(float) * nvals * rows);
    o.strip_partial[s] = take(sizeof(double) * nvals * strips);
  }
  for (int s = 0; s < L.nseg; ++s) o.squads[s] = take(sizeof(SquadState) * L.seg[s].nsquads);
  o.counters = take(sizeof(SquadState));
  o.ring = take(sizeof(int) * (size_t)npairs);
  o.bytes = at;
  return o;
}

// The launch plan (launch_plan.h) of a match over levels first .. last of npairs pairs shaped like `ref`, on the grid of v's
// instances, with the plan overrides of the environment as they are now.
LaunchPlan plan_launches(const dvo_b200_ctx* ctx, const dvo_b200_pyramid* ref, int first, int last, int npairs, const LevelVariant& v) {
  LevelShape shape[kMaxLevels];
  for (int l = 0; l <= first; ++l) shape[l] = {ref->L[l].h, ref->L[l].nbands, ref->L[l].nstrips};
  return make_launch_plan(shape, first, last, grid_ctas(ctx, v), npairs, plan_knobs_from_env());
}

// One run of the level kernel over pyramid levels first .. last of npairs pairs, pair q being (refs[q], curs[q]): the pairs
// of a match, or the virtual pairs of a multi-hypothesis screening.  A call's legs run in order, each taking its pair slots
// (states, iteration logs), descriptors ([level][pair], inside ws.d_pair_level, whose index CurPairLevel::csat shares) and
// level-flag slots after those of the leg before it.  li0 is the position of its first level in Result.Statistics.Levels: a
// leg that starts the pairs from T_init has li0 = 0, a later one continues the pairs the leg before it chose.  A leg with
// first < last runs no level; it only holds the pair slots of a continuation, and with maps_desc the descriptors of level
// `last` of its pairs, which the weight maps read.
struct Leg {
  int first, last, npairs;
  dvo_b200_pyramid* const* refs;
  dvo_b200_pyramid* const* curs;
  LaunchPlan plan;
  size_t pair0, desc0, ndesc;
  int li0, flag0;
};

Leg make_leg(const dvo_b200_ctx* ctx, const Leg* before, int first, int last, int npairs, dvo_b200_pyramid* const* refs,
             dvo_b200_pyramid* const* curs, const LevelVariant& v, bool maps_desc = false) {
  Leg g{first, last, npairs, refs, curs, {}, 0, 0, (size_t)npairs * std::max(first - last + 1, maps_desc ? 1 : 0), 0, 0};
  if (first >= last) g.plan = plan_launches(ctx, refs[0], first, last, npairs, v);
  if (before) {
    g.pair0 = before->pair0 + before->npairs; g.desc0 = before->desc0 + before->ndesc;
    g.li0 = before->li0 + before->first - before->last + 1; g.flag0 = before->flag0 + before->plan.nlaunch;
  }
  return g;
}

// The workspace of a call's legs: the descriptors, current-mask summaries, states and iteration logs of all of them, the
// scratch arena of their largest launch, the initial estimates of the first leg's pairs, the (alpha, beta) states and priors
// of the pairs, the residual-record dump of the test hook and the level flags.
int ensure_workspace(dvo_b200_ctx* ctx, const Leg* legs, int nlegs, size_t dump_floats, int max_log, const LevelVariant& v) {
  Workspace& ws = ctx->ws;
  const Leg& z = legs[nlegs - 1];
  const size_t ndesc = z.desc0 + z.ndesc, npairs = z.pair0 + z.npairs;
  const int nvals = v.affine ? kNormalValuesAffine : kNormalValues;
  size_t scratch = 0;
  for (int j = 0; j < nlegs; ++j)
    for (int i = 0; i < legs[j].plan.nlaunch; ++i)
      scratch = std::max(scratch, scratch_layout(legs[j].plan.launch[i], legs[j].npairs, nvals).bytes);
  int rc;
  if ((rc = grow(ctx, ws.d_pair_level, ws.cap_pair_level, ndesc + 1))) return rc;   // + 1: slack for whole 16-byte words
  if (v.cur_mask && (rc = grow(ctx, ws.d_csat, ws.cap_csat, ndesc + 1))) return rc;
  if ((rc = grow(ctx, ws.d_state, ws.cap_state, npairs))) return rc;
  if (max_log > 0 && (rc = grow(ctx, ws.d_iter_log, ws.cap_iter_log, npairs * max_log))) return rc;
  if ((rc = grow(ctx, ws.d_tinit, ws.cap_tinit, (size_t)16 * legs[0].npairs))) return rc;
  if (v.affine && (rc = grow(ctx, ws.d_affine, ws.cap_affine, npairs))) return rc;
  if (v.prior && (rc = grow(ctx, ws.d_prior, ws.cap_prior, (size_t)36 * npairs))) return rc;
  if ((rc = grow(ctx, ws.d_scratch, ws.cap_scratch, scratch))) return rc;
  if ((rc = grow(ctx, ws.d_dump, ws.cap_dump, dump_floats))) return rc;
  if (!ws.h_active) DVO_CUDA(ctx, cudaMallocHost((void**)&ws.h_active, sizeof(int) * kMaxLevels));
  return 0;
}

// One pyramid of each distinct slab among the batch's pyramids (a batch built in one call shares one slab), in slab order.
std::vector<const dvo_b200_pyramid*> distinct_slabs(int n, dvo_b200_pyramid* const* refs, dvo_b200_pyramid* const* curs) {
  std::vector<const dvo_b200_pyramid*> v;
  v.reserve(2 * (size_t)n);
  for (int i = 0; i < n; ++i) { v.push_back(refs[i]); v.push_back(curs[i]); }
  std::sort(v.begin(), v.end(), [](const dvo_b200_pyramid* a, const dvo_b200_pyramid* b) { return std::less<Slab*>()(a->slab, b->slab); });
  v.erase(std::unique(v.begin(), v.end(), [](const dvo_b200_pyramid* a, const dvo_b200_pyramid* b) { return a->slab == b->slab; }), v.end());
  return v;
}

int check_batch(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int n, dvo_b200_pyramid* const* refs,
                dvo_b200_pyramid* const* curs) {
  if (!cfg || n <= 0 || !refs || !curs) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match: null argument");
  if (cfg->first_level < cfg->last_level || cfg->last_level < 0 || cfg->first_level >= kMaxLevels)
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match: config not sane (FirstLevel >= LastLevel >= 0 required)");
  if (cfg->max_iterations_per_level < 0) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match: max iterations < 0");
  for (int i = 0; i < n; ++i) {
    if (!refs[i] || !curs[i]) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match: null pyramid");
    if (refs[i]->levels <= cfg->first_level || curs[i]->levels <= cfg->first_level)
      return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match: pyramid has fewer levels than FirstLevel+1");
    if (refs[i]->L[0].w != refs[0]->L[0].w || refs[i]->L[0].h != refs[0]->L[0].h ||
        curs[i]->L[0].w != refs[0]->L[0].w || curs[i]->L[0].h != refs[0]->L[0].h)
      return set_error(ctx, DVO_B200_ERR_SHAPE_MISMATCH, "match: all pyramids of a batch must share width/height");
  }
  // order this stream after the builds (possibly on another ctx's stream, possibly still running) of every pyramid
  for (const dvo_b200_pyramid* p : distinct_slabs(n, refs, curs)) wait_for_pyramid(ctx, p);
  return 0;
}

// After enqueueing a call's work on the batch: surface a launch error, remember the work on every slab of another context
// (Slab::foreign_uses; the caller may release the pyramids once the call returns), and leave the call's nflags level flags
// to the next synchronisation point (check_level_flags).
int end_call(dvo_b200_ctx* ctx, int n, dvo_b200_pyramid* const* refs, dvo_b200_pyramid* const* curs, int nflags) {
  DVO_CUDA(ctx, cudaGetLastError());
  for (const dvo_b200_pyramid* p : distinct_slabs(n, refs, curs))
    if (int rc = note_foreign_use(ctx, p)) return rc;
  ctx->pending_level_flags = nflags;
  return 0;
}

// The descriptors of n pairs at one level, and with csat their CurPairLevel::csat (kCurMask launches)
void fill_pair_levels(PairLevel* h, const int** csat, int n, dvo_b200_pyramid* const* refs, dvo_b200_pyramid* const* curs,
                      int level) {
  for (int i = 0; i < n; ++i) {
    const dvo_b200_pyramid* r = refs[i];
    const dvo_b200_pyramid* c = curs[i];
    const LevelInfo& rl = r->L[level];
    const LevelInfo& cl = c->L[level];
    PairLevel& q = h[i];
    const size_t plane = (size_t)rl.pitch * rl.h;
    q.r0 = r->planes + rl.rec_off; q.rp0 = r->planes + rl.plane_off;
    q.rmask = r->sel_mask + rl.mask_off;
    q.rsel = r->sel_info + 2 * level;
    q.rtmpl = r->tmpl + rl.tmpl_off;
    q.rrange = r->tile_range + rl.range_off;
    q.c0 = c->planes + cl.plane_off; q.c3 = q.c0 + plane;
    q.cfx = cl.fx; q.cfy = cl.fy; q.cox = cl.ox; q.coy = cl.oy;
    // PointSelection::getMaximumNumberOfPoints (point_selection.cpp:68-71)
    q.max_valid_pixels = (long long)(size_t)((double)r->L[0].n * pow(0.25, (double)level));
    if (csat) csat[i] = c->cur_sat ? c->cur_sat + cl.sat_off : nullptr;
  }
}

// The level kernel instance with the current-role mask test: iff some pair's current pyramid has a mask in that role.
bool any_current_mask(int n, dvo_b200_pyramid* const* curs) {
  for (int i = 0; i < n; ++i)
    if (curs[i]->cur_sat) return true;
  return false;
}

// The start of a call on the n pairs (refs[i], curs[i]) that check_batch passed: its level kernel instance v, that
// instance's grid, and the point selection of every reference at cfg's thresholds (PointSelection caches per pyramid,
// point_selection.cpp:100-113).
int begin_call(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int n, dvo_b200_pyramid* const* refs, dvo_b200_pyramid* const* curs,
               bool affine, bool prior, LevelVariant& v) {
  v = {ctx->estimator == DVO_B200_ESTIMATOR_CORRECTED, any_current_mask(n, curs), affine, prior};
  int rc = ensure_geometry(ctx, v);
  for (int i = 0; i < n && !rc; ++i)
    rc = pyramid_reselect(ctx, refs[i], cfg->intensity_derivative_threshold, cfg->depth_derivative_threshold);
  return rc;
}

LevelLaunch make_level_launch(const LevelInfo& L, const dvo_b200_config* cfg, int li, int level) {
  LevelLaunch lp;
  lp.w = L.w; lp.h = L.h; lp.n = L.n; lp.pitch = L.pitch; lp.nbands = L.nbands; lp.nstrips = L.nstrips;
  lp.level_index = li; lp.level_id = level; lp.max_iterations = cfg->max_iterations_per_level;
  lp.first_level = li == 0; lp.use_initial_estimate = cfg->use_initial_estimate;
  lp.precision = cfg->precision; lp.mu = cfg->mu;
  return lp;
}

// Enqueue launch i of leg g, whose level li is pyramid level g.first - li of the leg's pairs and level g.li0 + li of the match.
// Squad states, queues, the ready ring and the error flag are zeroed first; the error flag is copied to
// ws.h_active[g.flag0 + i] after the launch.  d_Tinit: the initial estimates of the leg's pairs (device memory) or NULL.
int launch_segments(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, const Leg& g, int i, const double* d_Tinit, int max_log,
                    float* dump, int skip_begin, const LevelVariant& v) {
  Workspace& ws = ctx->ws;
  cudaStream_t st = ctx->stream;
  const PlanLaunch& L = g.plan.launch[i];
  const int index = g.flag0 + i, npairs = g.npairs, first = g.first;
  const LevelInfo* const levels = g.refs[0]->L;
  const ScratchLayout o = scratch_layout(L, npairs, v.affine ? kNormalValuesAffine : kNormalValues);
  char* const base = ws.d_scratch;
  DVO_CUDA(ctx, cudaMemsetAsync(base + o.squads[0], 0, o.bytes - o.squads[0], st));
  PersistentArgs pa;
  pa.states = ws.d_state + g.pair0;
  int* counters = reinterpret_cast<int*>(base + o.counters);
  pa.error_flag = counters + 3 * kMaxSeg;
  pa.ilog = ws.d_iter_log + g.pair0 * max_log; pa.max_log = max_log;
  pa.T_init = d_Tinit; pa.skip_begin = skip_begin;
  pa.dump = dump;
  pa.npairs = npairs; pa.nseg = L.nseg;
  pa.pls0 = ws.d_pair_level; pa.csat = ws.d_csat;
  pa.affine = v.affine ? ws.d_affine + g.pair0 : nullptr;      // the per-pair mode state, in the leg's pair slots like the states
  pa.prior = v.prior ? ws.d_prior + 36 * g.pair0 : nullptr;
  for (int s = 0; s < L.nseg; ++s) {
    const PlanSegment& P = L.seg[s];
    Segment& S = pa.seg[s];
    S.pls = ws.d_pair_level + g.desc0 + (size_t)P.first_li * npairs;
    S.row_exports = reinterpret_cast<float*>(base + o.row_exports[s]);
    S.row_base = reinterpret_cast<int*>(base + o.row_base[s]);
    S.strip_exports = reinterpret_cast<double*>(base + o.strip_exports[s]);
    S.strip_base = reinterpret_cast<int*>(base + o.strip_base[s]);
    S.row_partial = reinterpret_cast<float*>(base + o.row_partial[s]);
    S.strip_partial = reinterpret_cast<double*>(base + o.strip_partial[s]);
    S.squads = reinterpret_cast<SquadState*>(base + o.squads[s]);
    S.queue = counters + s; S.ready_tail = counters + kMaxSeg + s; S.arrivals = counters + 2 * kMaxSeg + s;
    S.ready = reinterpret_cast<int*>(base + o.ring) + P.pair_begin;
    S.cyclic = P.cyclic; S.pair_begin = P.pair_begin; S.npairs_seg = P.npairs;
    S.dbg = ctx->d_dbg ? ctx->d_dbg + 16 * (index + s) : nullptr;
    S.dbg2 = ctx->d_dbg ? ctx->d_dbg + 128 + 8 * (index + s) : nullptr;
    S.nlev = P.nlev; S.g = P.g; S.nsquads = P.nsquads;
    for (int k = 0; k < kMaxLevels; ++k) S.strips_per_cta[k] = P.strips_per_cta[k];
    for (int k = 0; k < P.nlev; ++k) {
      const int li = P.first_li + k;
      S.lp[k] = make_level_launch(levels[first - li], cfg, g.li0 + li, first - li);
    }
  }
  {
    ProfScope prof(ctx, 0);
    ProfScope prof_level(ctx, 8 + index);
    void* args[] = {&pa};
    const LevelInstance li = level_instance(v);
    DVO_CUDA(ctx, cudaLaunchCooperativeKernel(li.kernel, dim3(grid_ctas(ctx, v)), dim3(kCtaThreads), args, li.smem, st));
    ctx->launches++;
  }
  DVO_CUDA(ctx, cudaMemcpyAsync(&ws.h_active[index], pa.error_flag, sizeof(int), cudaMemcpyDeviceToHost, st));
  return 0;
}

// The pinned stage of a call, in 16-byte aligned sections: ndesc pair descriptors (those of every level, [level][pair]), the
// initial estimates of n pairs (a test hook's T), the current-mask summaries (CurPairLevel::csat, same index as the
// descriptors), (alpha, beta) and the prior informations of n pairs.  A section the call does not need has 0 bytes.  `bytes` is what crosses PCIe: whole
// 16-byte words for the sections k_stage_words copies, and the doubles themselves for (alpha, beta), which k_affine_init
// reads in place.
struct MatchStageLayout {
  struct Section { size_t at, bytes; };
  Section desc, tinit, csat, ab, prior;
  size_t total;
};

MatchStageLayout match_stage_layout(size_t ndesc, int n, bool have_init, bool have_ab, const LevelVariant& v) {
  auto words = [](size_t bytes) { return (bytes + 15) / 16 * 16; };
  MatchStageLayout s;
  size_t at = 0;
  auto take = [&](size_t bytes) { const MatchStageLayout::Section o{at, bytes}; at += words(bytes); return o; };
  s.desc = take(words(sizeof(PairLevel) * ndesc));
  s.tinit = take(have_init ? sizeof(double) * 16 * (size_t)n : 0);
  s.csat = take(v.cur_mask ? words(sizeof(const int*) * ndesc) : 0);
  s.ab = take(have_ab ? sizeof(double) * 2 * (size_t)n : 0);
  s.prior = take(v.prior ? sizeof(double) * 36 * (size_t)n : 0);
  s.total = at;
  return s;
}

// Enqueue the copy of `bytes` (whole 16-byte words) of the pinned stage at `src` to device memory by k_stage_words.
void stage_words(dvo_b200_ctx* ctx, const void* src, void* dst, size_t bytes) {
  const size_t n16 = bytes / 16;
  k_stage_words<<<(unsigned)((n16 + 255) / 256), 256, 0, ctx->stream>>>((const uint4*)src, (uint4*)dst, n16);
  ctx->launches++;
}

// Stage a call's inputs once the previous use of the pinned stage and of the level flags has drained: the descriptors (and
// current-mask summaries) of every leg's levels, and for the pairs of the first leg the initial estimates T, (alpha, beta)
// ab of the photometric mode (NULL = (1, 0) each) and the prior informations, each NULL if the call has none.  The stage is
// copied to device memory by one small kernel per section (reads over PCIe: no H2D copy-engine work, no host round trip
// before the launches).  Then the level flags and the iteration logs of every leg start at zero.
int stage_inputs(dvo_b200_ctx* ctx, const Leg* legs, int nlegs, const double* T, const double* ab, const double* prior,
                 int max_log, const LevelVariant& v) {
  Workspace& ws = ctx->ws;
  cudaStream_t st = ctx->stream;
  const Leg& z = legs[nlegs - 1];
  const int n = legs[0].npairs;
  const MatchStageLayout s = match_stage_layout(z.desc0 + z.ndesc, n, T != nullptr, ab != nullptr, v);
  if (int rc = ensure_stage(ctx, 0, s.total)) return rc;
  DVO_CUDA(ctx, cudaStreamSynchronize(st));
  char* const h = (char*)ctx->h_stage;
  PairLevel* const h_desc = (PairLevel*)(h + s.desc.at);
  const int** h_csat = (const int**)(h + s.csat.at);
  for (int j = 0; j < nlegs; ++j) {
    const Leg& g = legs[j];
    // a leg that runs no level and has descriptors (make_leg's maps_desc) holds those of level g.last
    const int top = g.first < g.last && g.ndesc ? g.last : g.first;
    for (int level = top, li = 0; level >= g.last; --level, ++li) {
      const size_t at = g.desc0 + (size_t)li * g.npairs;
      fill_pair_levels(h_desc + at, v.cur_mask ? h_csat + at : nullptr, g.npairs, g.refs, g.curs, level);
    }
  }
  if (s.tinit.bytes) std::memcpy(h + s.tinit.at, T, s.tinit.bytes);
  if (s.ab.bytes) std::memcpy(h + s.ab.at, ab, s.ab.bytes);
  if (s.prior.bytes) std::memcpy(h + s.prior.at, prior, s.prior.bytes);
  ctx->h2d_bytes += s.desc.bytes + s.tinit.bytes + s.csat.bytes + s.ab.bytes + s.prior.bytes;
  {
    ProfScope prof(ctx, 2);
    stage_words(ctx, h_desc, ws.d_pair_level, s.desc.bytes);
    if (s.tinit.bytes) stage_words(ctx, h + s.tinit.at, ws.d_tinit, s.tinit.bytes);
    if (v.cur_mask) stage_words(ctx, h_csat, ws.d_csat, s.csat.bytes);
    if (v.affine) {
      k_affine_init<<<(n + 255) / 256, 256, 0, st>>>(ws.d_affine, s.ab.bytes ? (const double*)(h + s.ab.at) : nullptr, n);
      ctx->launches++;
    }
    if (v.prior) stage_words(ctx, h + s.prior.at, ws.d_prior, s.prior.bytes);
  }
  for (int i = 0; i < kMaxLevels; ++i) ws.h_active[i] = 0;
  if (max_log > 0)
    DVO_CUDA(ctx, cudaMemsetAsync(ws.d_iter_log, 0, sizeof(dvo_b200_iteration_stats) * (z.pair0 + z.npairs) * max_log, st));
  return 0;
}

// Enqueue the result assembly of n pair states into device memory
void finalize(dvo_b200_ctx* ctx, PairState* states, dvo_b200_result* d_res, int n) {
  ProfScope prof(ctx, 2);
  k_finalize<<<(n + 63) / 64, 64, 0, ctx->stream>>>(states, d_res, n);
  ctx->launches++;
}

// ctx->h_results of at least `bytes`: the pinned buffer the results of a call are copied back through
int ensure_pinned_results(dvo_b200_ctx* ctx, size_t bytes) {
  if (bytes > ctx->h_results_bytes) {
    if (ctx->h_results) cudaFreeHost(ctx->h_results);
    ctx->h_results = nullptr; ctx->h_results_bytes = 0;
    DVO_CUDA(ctx, cudaMallocHost(&ctx->h_results, bytes));
    ctx->h_results_bytes = bytes;
  }
  return 0;
}

// Enqueue the copy of (alpha, beta) of the n brightness states at src to dst, 2 n doubles of the pinned results buffer
int copy_back_photometric(dvo_b200_ctx* ctx, void* dst, const AffineState* src, size_t n) {
  DVO_CUDA(ctx, cudaMemcpy2DAsync(dst, 2 * sizeof(double), src->ab, sizeof(AffineState), 2 * sizeof(double), n,
                                  cudaMemcpyDeviceToHost, ctx->stream));
  return 0;
}

}  // namespace

// A match (k = 0) is one leg over levels first .. last of the n pairs.  A multi-hypothesis match (include/dvo_b200.h) is two:
// the screening leg runs n k virtual pairs, pair p k + j being (refs[p], curs[p]) from H[p][j] (and Lambda[p][j],
// (alpha, beta)_0[p][j]), on levels first .. s; k_pick_hypotheses scores them and copies each pair's chosen state (log,
// AffineState, Lambda) into its slot of the continuation leg, which runs levels s-1 .. last (none if s = last) on the n
// chosen pairs, its level indices continuing at first - s + 1.  Both legs launch the level kernel like any other match, so
// plan independence gives each pair the bits of one plain match of its mode.  With maps the continuation leg also holds the
// level-last descriptors of its pairs when it runs no level (s = last), so that k_weight_maps reads the descriptors, states
// and AffineStates of the last leg whichever the call.  The device stage holds the results (n), screen results (n k, if
// requested), scores (n k) and best (n; none of the three with k = 0), copied back through the pinned results buffer in
// that layout, followed there at the next 16-byte boundary by (alpha, beta) of the n pairs and of the n k screening runs
// (if requested).  A device-results call writes its results to d_results and uses neither.
int tracker_match(dvo_b200_ctx* ctx, const MatchCall& c) {
  const dvo_b200_config* const cfg = c.cfg;
  dvo_b200_pyramid* const* const refs = c.refs;
  dvo_b200_pyramid* const* const curs = c.curs;
  int rc = check_batch(ctx, cfg, c.n, refs, curs);
  if (rc) return rc;
  LevelVariant v;
  if ((rc = begin_call(ctx, cfg, c.n, refs, curs, c.ab_out != nullptr, c.prior != nullptr, v))) return rc;
  cudaStream_t st = ctx->stream;
  Workspace& ws = ctx->ws;
  const int n = c.n, k = c.k, nk = n * k, last = cfg->last_level;
  const int max_log = c.iter_stats ? c.max_log : 0;
  std::vector<dvo_b200_pyramid*> vrefs((size_t)nk), vcurs((size_t)nk);
  for (int q = 0; q < nk; ++q) { vrefs[q] = refs[q / k]; vcurs[q] = curs[q / k]; }
  Leg legs[2];
  const int nlegs = k ? 2 : 1;
  if (k) {
    legs[0] = make_leg(ctx, nullptr, cfg->first_level, c.screen_level, nk, vrefs.data(), vcurs.data(), v);
    legs[1] = make_leg(ctx, &legs[0], c.screen_level - 1, last, n, refs, curs, v, c.maps != nullptr);
  } else {
    legs[0] = make_leg(ctx, nullptr, cfg->first_level, last, n, refs, curs, v);
  }
  const Leg& z = legs[nlegs - 1];   // the leg the results come from
  if ((rc = ensure_workspace(ctx, legs, nlegs, 0, max_log, v))) return rc;
  if (c.maps && (rc = weight_maps_prepare(ctx, *c.maps, n, refs[0], last))) return rc;

  const size_t res_bytes = sizeof(dvo_b200_result) * (size_t)n;
  const size_t screen_bytes = c.screen_results ? sizeof(dvo_b200_result) * (size_t)nk : 0, score_bytes = sizeof(double) * (size_t)nk;
  const size_t scores_at = res_bytes + screen_bytes, best_at = scores_at + score_bytes;
  const size_t out_bytes = best_at + (k ? sizeof(int32_t) * (size_t)n : 0);
  const size_t ab_at = (out_bytes + 15) / 16 * 16, ab_bytes = v.affine ? sizeof(double) * 2 * (size_t)n : 0;
  const size_t screen_ab_bytes = c.screen_ab ? sizeof(double) * 2 * (size_t)nk : 0;
  if (!c.d_results) {
    if ((rc = ensure_stage(ctx, out_bytes, 0))) return rc;
    if ((rc = ensure_pinned_results(ctx, ab_at + ab_bytes + screen_ab_bytes))) return rc;
  }
  const double* const tinit = cfg->use_initial_estimate ? c.T_init : nullptr;
  if ((rc = stage_inputs(ctx, legs, nlegs, tinit, c.ab_init, c.prior, max_log, v))) return rc;
  for (int i = 0; i < legs[0].plan.nlaunch; ++i)
    if ((rc = launch_segments(ctx, cfg, legs[0], i, tinit ? ws.d_tinit : nullptr, max_log, nullptr, 0, v))) return rc;
  char* const d_out = (char*)ctx->d_stage;
  dvo_b200_result* const d_res = c.d_results ? (dvo_b200_result*)c.d_results : (dvo_b200_result*)d_out;
  if (k) {
    const Leg &screen = legs[0], &chosen = legs[1];
    if (c.screen_results) finalize(ctx, ws.d_state, (dvo_b200_result*)(d_out + res_bytes), nk);
    {
      ProfScope prof(ctx, 2);
      auto pick = v.affine ? (v.prior ? k_pick_hypotheses<true, true> : k_pick_hypotheses<true, false>)
                           : (v.prior ? k_pick_hypotheses<false, true> : k_pick_hypotheses<false, false>);
      pick<<<(n + 3) / 4, 128, 0, st>>>(ws.d_state, ws.d_iter_log, ws.d_state + chosen.pair0, ws.d_iter_log + chosen.pair0 * max_log,
                                        max_log, n, k, screen.first - screen.last, c.min_ratio, (double*)(d_out + scores_at),
                                        (int*)(d_out + best_at), v.affine ? ws.d_affine : nullptr,
                                        v.affine ? ws.d_affine + chosen.pair0 : nullptr, v.prior ? ws.d_prior : nullptr,
                                        v.prior ? ws.d_prior + 36 * chosen.pair0 : nullptr);
      ctx->launches++;
    }
    for (int i = 0; i < chosen.plan.nlaunch; ++i)
      if ((rc = launch_segments(ctx, cfg, chosen, i, nullptr, max_log, nullptr, 0, v))) return rc;
  }
  finalize(ctx, ws.d_state + z.pair0, d_res, n);
  if (c.maps)
    weight_maps_launch(ctx, *c.maps, n, refs[0], last, ws.d_state + z.pair0, ws.d_pair_level + z.desc0 + z.ndesc - n,
                       v.affine ? ws.d_affine + z.pair0 : nullptr);
  if ((rc = end_call(ctx, n, refs, curs, z.flag0 + z.plan.nlaunch))) return rc;
  if (c.d_results) return 0;   // a device-results call leaves its level flags to dvo_b200_synchronize

  char* const hr = (char*)ctx->h_results;
  const size_t log_bytes = sizeof(dvo_b200_iteration_stats) * (size_t)n * max_log;
  DVO_CUDA(ctx, cudaMemcpyAsync(hr, d_out, out_bytes, cudaMemcpyDeviceToHost, st));
  if (ab_bytes && (rc = copy_back_photometric(ctx, hr + ab_at, ws.d_affine + z.pair0, (size_t)n))) return rc;
  if (screen_ab_bytes && (rc = copy_back_photometric(ctx, hr + ab_at + ab_bytes, ws.d_affine, (size_t)nk))) return rc;
  if (c.maps && (rc = weight_maps_copy_back(ctx, *c.maps, n, refs[0], last))) return rc;
  if (log_bytes)
    DVO_CUDA(ctx, cudaMemcpyAsync(c.iter_stats, ws.d_iter_log + z.pair0 * max_log, log_bytes, cudaMemcpyDeviceToHost, st));
  ctx->d2h_bytes += out_bytes + ab_bytes + screen_ab_bytes + log_bytes;
  DVO_CUDA(ctx, cudaStreamSynchronize(st));
  std::memcpy(c.results, hr, res_bytes);
  if (screen_bytes) std::memcpy(c.screen_results, hr + res_bytes, screen_bytes);
  if (c.scores) std::memcpy(c.scores, hr + scores_at, score_bytes);
  if (k) std::memcpy(c.best, hr + best_at, out_bytes - best_at);
  if (ab_bytes) std::memcpy(c.ab_out, hr + ab_at, ab_bytes);
  if (screen_ab_bytes) std::memcpy(c.screen_ab, hr + ab_at + ab_bytes, screen_ab_bytes);
  return check_level_flags(ctx);
}

// The persistent kernels report a barrier / transaction timeout through a flag copied to pinned memory after every level.
// Call after the stream has been synchronised.
int check_level_flags(dvo_b200_ctx* ctx) {
  Workspace& ws = ctx->ws;
  const int nl = ctx->pending_level_flags;
  ctx->pending_level_flags = 0;
  if (!ws.h_active) return 0;
  for (int li = 0; li < nl && li < kMaxLevels; ++li)
    if (ws.h_active[li] != 0) {
      const int code = ws.h_active[li];
      ws.h_active[li] = 0;
      return set_error(ctx, DVO_B200_ERR_CUDA, code == 2 ? "persistent level kernel: bulk-copy transaction timed out"
                                                         : "persistent level kernel: squad barrier timed out");
    }
  return 0;
}

// Test hooks (dvo_b200_residual_image, dvo_b200_linearize): ONE Gauss-Newton iteration of the level kernel for one
// pair at a fixed transform: stage A, P_k, stage B (optionally dumping the residual records), end step.  The pair's leg
// is staged like a match with T as its initial estimate, which k_set_state places into the state.
int tracker_linearize(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* ref, dvo_b200_pyramid* cur,
                      int level, const double* T, int use_weights, const float* prev_precision, int64_t* count,
                      float* precision_out, float* ll_out, double* A_out, double* b_out, float* planes7, const double* ab) {
  dvo_b200_config c = *cfg;
  c.first_level = level; c.last_level = level;
  dvo_b200_pyramid* refs[1] = {ref};
  dvo_b200_pyramid* curs[1] = {cur};
  int rc = check_batch(ctx, &c, 1, refs, curs);
  if (rc) return rc;
  if (!T) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "linearize: T is null");
  LevelVariant v;
  if ((rc = begin_call(ctx, cfg, 1, refs, curs, ab != nullptr, false, v))) return rc;
  cudaStream_t st = ctx->stream;
  Workspace& ws = ctx->ws;
  const LevelInfo& L = ref->L[level];
  const Leg leg = make_leg(ctx, nullptr, level, level, 1, refs, curs, v);
  if ((rc = ensure_workspace(ctx, &leg, 1, planes7 ? 7 * (size_t)L.n : 0, 0, v))) return rc;
  c.max_iterations_per_level = use_weights ? 2 : 1;    // k_set_state starts at iteration 1 / 0: exactly one iteration runs
  c.use_initial_estimate = 0; c.precision = 0.0; c.mu = 0.0;
  if ((rc = stage_inputs(ctx, &leg, 1, T, ab, nullptr, 0, v))) return rc;
  const float* pp = use_weights ? prev_precision : nullptr;
  k_set_state<<<1, 1, 0, st>>>(ws.d_state, ws.d_pair_level, ws.d_tinit, pp ? make_float4(pp[0], pp[1], pp[2], pp[3]) : float4{},
                               use_weights, make_level_launch(L, &c, 0, level));
  ctx->launches += 1;
  for (int i = 0; i < leg.plan.nlaunch; ++i)
    if ((rc = launch_segments(ctx, &c, leg, i, nullptr, 0, planes7 ? ws.d_dump : nullptr, 1, v))) return rc;
  if ((rc = end_call(ctx, 1, refs, curs, leg.plan.nlaunch))) return rc;
  const size_t affine_at = (sizeof(PairState) + 15) / 16 * 16;   // the pinned results: the pair's state, then its AffineState
  if ((rc = ensure_pinned_results(ctx, affine_at + sizeof(AffineState)))) return rc;
  PairState* const hs = (PairState*)ctx->h_results;
  AffineState* const ha = (AffineState*)((char*)ctx->h_results + affine_at);
  DVO_CUDA(ctx, cudaMemcpyAsync(hs, ws.d_state, sizeof(PairState), cudaMemcpyDeviceToHost, st));
  if (v.affine) DVO_CUDA(ctx, cudaMemcpyAsync(ha, ws.d_affine, sizeof(AffineState), cudaMemcpyDeviceToHost, st));
  DVO_CUDA(ctx, cudaStreamSynchronize(st));
  if ((rc = check_level_flags(ctx))) return rc;
  if (count) *count = hs->n;
  if (precision_out) std::memcpy(precision_out, hs->precision, sizeof(float) * 4);
  if (ll_out) *ll_out = hs->ll;
  if (A_out) std::memcpy(A_out, v.affine ? ha->A : hs->A, sizeof(double) * (v.affine ? 64 : 36));
  if (b_out) std::memcpy(b_out, v.affine ? ha->b : hs->b, sizeof(double) * (v.affine ? 8 : 6));
  if (planes7) {
    // {ei, ez, gx, gy, hx, hy, z_ref}; invalid -> NaN in every plane
    DVO_CUDA(ctx, cudaMemcpy(planes7, ws.d_dump, sizeof(float) * 7 * (size_t)L.n, cudaMemcpyDeviceToHost));
    ctx->d2h_bytes += sizeof(float) * 7 * (size_t)L.n;
  }
  return 0;
}

}  // namespace dvo_b200
