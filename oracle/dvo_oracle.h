/*
 * dvo_oracle.h -- CPU ORACLE for the dvo::DenseTracker::match() hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load it.  The product
 * (dvo_slam_b200/) never includes, links or calls anything in oracle/.
 *
 * What it is: a dependency-free C++17 restatement of the reference algorithm
 * (tum-vision/dvo_slam @ d25b65bf, dvo_core).  Every function cites the reference
 * file:line it follows.  Nothing here is copied from the reference: the reference is
 * Eigen/OpenCV/Sophus code that cannot be compiled in this image (those libraries are
 * absent, see DESIGN.md), so the arithmetic is restated with plain arrays.
 *
 * PARITY PINNED against the reference's own object code (tests/test_reference_pin.py): the reference ships no tests,
 * golden vectors or fixtures for this path (SURVEY.md section 4 / 8c) and its build system cannot run here, but its
 * hot-path translation units dvo_core/src/{dense_tracking_impl,core/math_sse,core/intrinsic_matrix}.cpp compile unmodified
 * against header-only container stand-ins (oracle/ref_shim/, recipe: oracle/Makefile target `ref`, output oracle/_ref/).
 * FAITHFUL mode equals that object code (-O2: arithmetic in program order) BIT FOR BIT on every golden case: counts,
 * validity, every residual-record value, P, log-likelihood, A, b; whole alignments driven through the reference's
 * functions have identical control flow.  What remains restated without a reference-side pin: the control flow of
 * dense_tracking.cpp (needs Sophus), the pyramid of rgbd_image.cpp (needs OpenCV proper), Sophus SE3 exp/log and Eigen's
 * LDLT -- pinned against analytic ground truth and closed-form identities (tests/test_oracle.py).
 *
 * Modes (orc_mode flags) -- each flag reproduces one numerical quirk of the reference:
 *   rcp_approx        _mm_rcp_ps in projection and weights   (dense_tracking_impl.cpp:192,700)
 *   rtz_residuals     MXCSR round-toward-zero in the residual loop (dense_tracking_impl.cpp:165-167)
 *   drop_odd_point    odd number of selected points -> last one skipped (dense_tracking_impl.cpp:169)
 *   scale_pair_bug    computeScaleSse adds w2*r1*r1^T for every pair (dense_tracking_impl.cpp:603-622)
 *   ll_drop_tail      log-likelihood drops the last n%50 terms (dense_tracking_impl.cpp:413-422)
 *   f32_serial_accum  fp32 strictly sequential A,b accumulation in the SSE block order
 *                     (least_squares.cpp:58-64, math_sse.cpp:82-178); off = fp64 accumulation
 *   fused_pixel_math  per-pixel arithmetic written with explicit fmaf() in the order the
 *                     CUDA kernels use (bit-mirror of the GPU residual record); off = the
 *                     reference's unfused mul/add order.
 *   ll_group_product  log-likelihood sum as the log of fp64 products of (1 + 0.2 d) over groups of 50 points
 *                     (dense_tracking_impl.cpp:406-425): a group whose product overflows makes it -inf, and the
 *                     iteration is rejected; off = the sum of the per-point logs, finite wherever every d is.
 * Presets: FAITHFUL = all reference quirks on, fused off.   (timed CPU baseline, parity target)
 *          EXACT    = everything off (exact division, nearest rounding, fp64 sums).
 *          MIRROR   = structural quirks on (drop_odd_point, scale_pair_bug, ll_drop_tail, ll_group_product),
 *                     numerical noise off, fused_pixel_math on: what the GPU path computes.
 *          The corrected estimator's definition (tests/helpers.py corrected_mode) is MIRROR with the four structural
 *          quirks off.
 */
#ifndef DVO_ORACLE_H_
#define DVO_ORACLE_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_MAX_LEVELS 8

typedef struct orc_mode {
  int rcp_approx;
  int rtz_residuals;
  int drop_odd_point;
  int scale_pair_bug;
  int ll_drop_tail;
  int f32_serial_accum;
  int fused_pixel_math;
  int ll_group_product;
} orc_mode;

/* mirrors dvo::DenseTracker::Config fields that influence match() (dense_tracking.h:42-69) */
typedef struct orc_config {
  int first_level;
  int last_level;
  int max_iterations_per_level;
  double precision;
  double mu;
  int use_initial_estimate;
  float intensity_derivative_threshold;
  float depth_derivative_threshold;
} orc_config;

/* dvo::DenseTracker::TerminationCriteria (dense_tracking.h:71-81) */
enum {
  ORC_TERM_ITERATIONS_EXCEEDED = 0,
  ORC_TERM_INCREMENT_TOO_SMALL = 1,
  ORC_TERM_LOG_LIKELIHOOD_DECREASED = 2,
  ORC_TERM_TOO_FEW_CONSTRAINTS = 3
};

/* dvo::DenseTracker::IterationStats (dense_tracking.h:83-101) */
typedef struct orc_iteration_stats {
  int32_t level;
  int32_t id;
  int64_t valid_constraints;
  double tdist_log_likelihood;   /* = -ll */
  double tdist_precision[4];     /* row-major 2x2 */
  double prior_log_likelihood;
  double increment[6];
  double information[36];        /* A incl. mu*I, row-major; NaN if never computed */
} orc_iteration_stats;

/* dvo::DenseTracker::LevelStats (dense_tracking.h:104-117) */
typedef struct orc_level_stats {
  int32_t id;
  int32_t termination;
  int64_t max_valid_pixels;
  int64_t valid_pixels;
  int32_t num_iterations;
  int32_t pad_;
} orc_level_stats;

/* dvo::DenseTracker::Result (dense_tracking.h:125-140) */
typedef struct orc_result {
  double transformation[16];     /* row-major 4x4, = estimate^-1 (dense_tracking.cpp:371) */
  double information[36];
  double log_likelihood;
  int32_t num_levels;
  int32_t pad_;
  orc_level_stats levels[ORC_MAX_LEVELS];
} orc_result;

typedef struct orc_pyramid orc_pyramid;

orc_mode orc_mode_faithful(void);
orc_mode orc_mode_exact(void);
orc_mode orc_mode_mirror(void);
orc_config orc_config_default(void);      /* dense_tracking_config.cpp:27-42 */

/* RgbdCameraPyramid(w,h,K)::create(intensity, depth) + RgbdImagePyramid::build(levels)
 * + derivatives (rgbd_image.cpp:156-172, 283-296, 419-472; rgbd_image_sse.cpp:241-284). */
orc_pyramid* orc_pyramid_create(const float* intensity, const float* depth, int width, int height,
                                float fx, float fy, float ox, float oy, int levels);
void orc_pyramid_destroy(orc_pyramid* p);
int orc_pyramid_num_levels(const orc_pyramid* p);
/* channel: 0 I, 1 Z, 2 Ix, 3 Iy, 4 Zx, 5 Zy.  Returns pointer to h*w floats. */
const float* orc_pyramid_plane(const orc_pyramid* p, int level, int channel);
void orc_pyramid_level_info(const orc_pyramid* p, int level, int* width, int* height, float K[4]);

/* PointSelection::select (point_selection.cpp:89-152).  mask may be NULL; else h*w bytes. */
int64_t orc_select(const orc_pyramid* ref, int level, float ti, float td, const orc_mode* mode,
                   uint8_t* mask);

/* One evaluation of computeResidualsSse at a given transform (dense_tracking_impl.cpp:133-393)
 * in dense image form: 7 planes of h*w floats {e.i, e.z, e.idx, e.idy, e.zdx, e.zdy, z_ref},
 * NaN in every plane where the reference point is not selected / not valid.  T is the 4x4
 * row-major double "estimate" (cast to float inside, dense_tracking.cpp:263).  ab: NULL, or the
 * photometric mode's (alpha, beta), applied to the reference intensities as alpha I_ref + beta
 * (float, rounded to nearest; fmaf under fused_pixel_math).  Returns n. */
int64_t orc_residual_image(const orc_pyramid* ref, const orc_pyramid* cur, int level,
                           const double T[16], const double ab[2], float ti, float td,
                           const orc_mode* mode, float* planes7);

/* DenseTracker::computeIntensityErrorImage (dense_tracking.cpp:378-444): h*w floats, |intensity residual| at
 * every selected pixel whose residual is valid, 0 elsewhere (including the odd last selected point, which the
 * SSE residual loop never visits).  Returns the number of residuals written. */
int64_t orc_intensity_error_image(const orc_pyramid* ref, const orc_pyramid* cur, int level,
                                  const double T[16], float ti, float td, const orc_mode* mode,
                                  float* image);

/* One full Gauss-Newton linearisation at T with given previous precision (iteration>0 semantics
 * when use_weights!=0, else weights=1): returns n, and fills scale precision P (row-major 2x2
 * float), ll (float), A (36 doubles incl. no mu), b (6 doubles).  Follows dense_tracking.cpp:271-343.
 * ab non-NULL: the photometric mode at (alpha, beta) as in orc_residual_image; A is then 8x8 (64
 * doubles) and b 8 doubles, the unknowns (pose, alpha, beta), with de_i/dalpha = -I_ref/255 and
 * de_i/dbeta = -1/255 on the intensity row. */
int64_t orc_linearize(const orc_pyramid* ref, const orc_pyramid* cur, int level, const double T[16],
                      const double ab[2], float ti, float td, int use_weights, const float prev_precision[4],
                      const orc_mode* mode, float precision_out[4], float* ll_out,
                      double* A_out, double* b_out);

/* DenseTracker::match(reference, current, result) (dense_tracking.cpp:123-376).
 * T_init: row-major 4x4 initial Result.Transformation (used iff cfg.use_initial_estimate).
 * iters: optional array of max_iters entries receiving every iteration of every level in order;
 * *num_iters receives the count.  Returns 0. */
int orc_match(orc_pyramid* ref, orc_pyramid* cur, const orc_config* cfg, const double T_init[16],
              const orc_mode* mode, orc_result* result, orc_iteration_stats* iters, int max_iters,
              int* num_iters);

/* orc_match with its optional inputs; orc_match is this with prior, ab_init and ab_out NULL.
 * prior: NULL, or a motion prior information Lambda (36 doubles, row-major) in place of cfg.mu I
 *   (cfg.mu is then ignored): A += Lambda and b += Lambda li on the pose block, and the prior
 *   log-likelihood li^T Lambda li, with li = log(initial).
 * ab_out: NULL, or the photometric mode, which receives the final (alpha, beta).  (alpha, beta) start
 *   at ab_init (NULL: (1, 0)) and are a Revertable updated with the pose: the top of every iteration
 *   adds the (alpha, beta) part of the level's last accepted increment, a rejected iteration reverts
 *   both, and levels carry them over.  The system is orc_linearize's 8x8 and the information its Schur
 *   complement onto the pose (prior included). */
int orc_match_with(orc_pyramid* ref, orc_pyramid* cur, const orc_config* cfg, const double T_init[16],
                   const double prior[36], const double ab_init[2], const orc_mode* mode, orc_result* result,
                   double ab_out[2], orc_iteration_stats* iters, int max_iters, int* num_iters);

/* SE(3) helpers (restated Sophus se3.hpp algorithm), exposed for tests. */
void orc_se3_exp(const double xi[6], double T[16]);
void orc_se3_log(const double T[16], double xi[6]);
/* Eigen-style pivoted LDLT solve of an n x n SPD system, n <= 8 (dense_tracking.cpp:347; n = 8 in the photometric mode). */
void orc_ldlt_solve(const double* A, const double* b, double* x, int n);
void orc_ldlt_solve6(const double A[36], const double b[6], double x[6]);   /* orc_ldlt_solve with n = 6 */
/* The Schur complement of an 8x8 onto its first 6 unknowns: the photometric mode's information. */
void orc_schur_onto_pose(const double A[64], double S[36]);

/* SurfacePyramid::convertRawDepthImageSse (surface_pyramid.cpp:45-105): u16 -> f32*scale, 0 -> NaN */
void orc_convert_raw_depth(const uint16_t* in, float* out, int64_t count, float scale);
/* cv::cvtColor(rgb, grey, CV_BGR2GRAY) on CV_8UC3 followed by convertTo(CV_32F) (call site benchmark_slam.cpp:58-68).
 * OpenCV (2.4.x, the version dvo_slam's rosbuild manifests pull in) is not vendored in the reference checkout; its published
 * 8-bit algorithm is fixed point: grey = (B*1868 + G*9617 + R*4899 + (1 << 13)) >> 14.  Known answers:
 * pure blue/green/red 255 -> 29/150/76, white -> 255. */
void orc_bgr_to_grey(const uint8_t* bgr, float* out, int64_t count);

#ifdef __cplusplus
}
#endif
#endif /* DVO_ORACLE_H_ */
