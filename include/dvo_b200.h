/*
 * dvo_b200.h -- C ABI of the CUDA-native (H100, sm_90a) dense RGB-D alignment engine.
 *
 * This is the drop-in boundary for ONE hot path of tum-vision/dvo_slam: dvo::DenseTracker::match()
 * (dvo_core/src/dense_tracking.cpp:123-376) and the image model it consumes
 * (dvo_core/src/core/rgbd_image.cpp, point_selection.cpp).  The reference has no FFI today: the
 * boundary there is the C++ class API of libdvo_core.so (dvo_core/include/dvo/dense_tracking.h:39-170,
 * dvo_core/include/dvo/core/rgbd_image.h:127-262).  The C++ adapter in include/dvo_b200/ keeps those
 * class signatures and forwards to the entry points below; INTEGRATION.md shows the binding.
 *
 * Plain C types only (no torch / Eigen / OpenCV types).  All functions return 0 on success and a
 * negative dvo_b200_status on failure; numerical failure is reported exactly like the reference
 * (NaN Result + TerminationCriterion), never as an error code (dense_tracking.cpp:135,375: match()
 * always returns true).  Nothing here falls back to a CPU implementation: without a CUDA device
 * dvo_b200_create fails with DVO_B200_ERR_CUDA.
 */
#ifndef DVO_B200_H_
#define DVO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DVO_B200_MAX_LEVELS 8
#define DVO_B200_ABI_VERSION 1

typedef enum dvo_b200_status {
  DVO_B200_OK = 0,
  DVO_B200_ERR_INVALID_ARGUMENT = -1,
  DVO_B200_ERR_CUDA = -2,
  DVO_B200_ERR_OUT_OF_MEMORY = -3,
  DVO_B200_ERR_SHAPE_MISMATCH = -4
} dvo_b200_status;

/* dvo::DenseTracker::TerminationCriteria::Enum (dense_tracking.h:71-81) -- same numeric values */
typedef enum dvo_b200_termination {
  DVO_B200_TERM_ITERATIONS_EXCEEDED = 0,
  DVO_B200_TERM_INCREMENT_TOO_SMALL = 1,
  DVO_B200_TERM_LOG_LIKELIHOOD_DECREASED = 2,
  DVO_B200_TERM_TOO_FEW_CONSTRAINTS = 3
} dvo_b200_termination;

/* The fields of dvo::DenseTracker::Config that match() reads (dense_tracking.h:42-69; defaults
 * dense_tracking_config.cpp:27-42).  UseWeighting / InfluenceFunction* / ScaleEstimator* /
 * UseParallel are accepted by the C++ adapter for API compatibility but never reach match() in the
 * reference either (dense_tracking.cpp:81-97 vs 286-295), so they are not part of the ABI. */
typedef struct dvo_b200_config {
  int32_t first_level;                  /* FirstLevel (coarsest), default 3 */
  int32_t last_level;                   /* LastLevel (finest), default 1 */
  int32_t max_iterations_per_level;     /* default 100 */
  int32_t use_initial_estimate;         /* default 0 */
  double precision;                     /* default 5e-7 */
  double mu;                            /* default 0 */
  float intensity_derivative_threshold; /* default 0 */
  float depth_derivative_threshold;     /* default 0 */
} dvo_b200_config;

/* dvo::DenseTracker::IterationStats (dense_tracking.h:83-101) */
typedef struct dvo_b200_iteration_stats {
  int32_t level;
  int32_t id;
  int64_t valid_constraints;
  double tdist_log_likelihood;          /* TDistributionLogLikelihood (= -ll, dense_tracking.cpp:299) */
  double tdist_precision[4];            /* row-major 2x2 */
  double prior_log_likelihood;
  double increment[6];                  /* EstimateIncrement; NaN if the iteration was rejected */
  double information[36];               /* EstimateInformation (A + mu*I), row-major; NaN if rejected */
} dvo_b200_iteration_stats;

/* dvo::DenseTracker::LevelStats (dense_tracking.h:104-117) plus what its helpers expose */
typedef struct dvo_b200_level_stats {
  int32_t id;
  int32_t termination;                  /* dvo_b200_termination */
  int64_t max_valid_pixels;             /* PointSelection::getMaximumNumberOfPoints (point_selection.cpp:68-71) */
  int64_t valid_pixels;                 /* number of selected reference points S */
  int32_t num_iterations;               /* Iterations.size() */
  int32_t has_iteration_with_increment; /* LevelStats::HasIterationWithIncrement (dense_tracking_config.cpp:138-143) */
  int64_t last_valid_constraints;       /* Iterations.back().ValidConstraints */
  /* LastIterationWithIncrement() (dense_tracking_config.cpp:145-155) is Iterations[size-2] after LogLikelihoodDecreased and
   * Iterations.back() after every other termination, TooFewConstraints included: then it is the entry with n < 6
   * constraints, whose log-likelihood is 0.  Both fields are -1 / NaN while has_iteration_with_increment is 0. */
  int64_t last_increment_valid_constraints; /* LastIterationWithIncrement().ValidConstraints, -1 if none */
  double last_increment_log_likelihood; /* LastIterationWithIncrement().TDistributionLogLikelihood, NaN if none */
} dvo_b200_level_stats;

/* dvo::DenseTracker::Result (dense_tracking.h:125-140) */
typedef struct dvo_b200_result {
  double transformation[16];            /* row-major 4x4; = estimate^-1 (dense_tracking.cpp:371) */
  double information[36];               /* row-major 6x6; = A_last * 0.008^2 (dense_tracking.cpp:372) */
  double log_likelihood;
  int32_t num_levels;
  int32_t num_iterations_total;
  dvo_b200_level_stats levels[DVO_B200_MAX_LEVELS];
} dvo_b200_result;

/* The estimator of the alignments on a context (dvo_b200_set_estimator).
 * REFERENCE (default): what dvo::DenseTracker::match() computes, including three structural quirks of its SSE code:
 *   the scale estimate adds w2 r1 r1^T instead of w2 r2 r2^T for every pair of points (dense_tracking_impl.cpp:614-615),
 *   the log-likelihood drops the last n mod 50 terms (dense_tracking_impl.cpp:413-422), and the last point of an odd
 *   selection is never visited (dense_tracking_impl.cpp:169).
 * CORRECTED: the same algorithm without those three: scale = sum_i w_i r_i r_i^T / (n - 3), the log-likelihood over all
 *   n points, and the odd last point is a constraint like any other.  Everything else is unchanged (Student-t weights with
 *   nu = 5 and P_{k-1}, the 1/(n-3) normaliser, the float log-likelihood, Jacobians at the untransformed point, the accept
 *   test, LDL^T, SE(3) update, termination; LevelStats.valid_pixels is still the selection count S).  Results differ from
 *   the reference's: this is for callers that want the estimator of the DVO papers, not a libdvo_core replacement. */
typedef enum dvo_b200_estimator {
  DVO_B200_ESTIMATOR_REFERENCE = 0,
  DVO_B200_ESTIMATOR_CORRECTED = 1
} dvo_b200_estimator;

typedef struct dvo_b200_ctx dvo_b200_ctx;          /* one per host thread / CUDA stream */
typedef struct dvo_b200_pyramid dvo_b200_pyramid;  /* device mirror of dvo::core::RgbdImagePyramid */

/* ---- context ------------------------------------------------------------------------------ */
int dvo_b200_abi_version(void);
/* device: CUDA ordinal.  stream: a cudaStream_t to run on, or NULL to create a private stream. */
int dvo_b200_create(int device, void* stream, dvo_b200_ctx** out);
int dvo_b200_destroy(dvo_b200_ctx* ctx);
void* dvo_b200_stream(dvo_b200_ctx* ctx);             /* the cudaStream_t all work is enqueued on */
int dvo_b200_synchronize(dvo_b200_ctx* ctx);
const char* dvo_b200_last_error(dvo_b200_ctx* ctx);   /* human readable, valid until next call */
void dvo_b200_config_default(dvo_b200_config* cfg);   /* DenseTracker::getDefaultConfig() */
/* counters for the bench harness: kernels launched / bytes copied through this ctx so far */
int64_t dvo_b200_kernel_launches(dvo_b200_ctx* ctx);
int64_t dvo_b200_h2d_bytes(dvo_b200_ctx* ctx);
int64_t dvo_b200_d2h_bytes(dvo_b200_ctx* ctx);
/* Estimator of every later call on ctx: match, match_batch[_device], and the test hooks residual_image, linearize and
 * intensity_error_image, which run the same kernel (in CORRECTED mode the odd last point appears in their outputs).  A
 * sharded caller sets it on each dvo_b200_sharded_ctx(s, i).  Pyramids are not touched: contexts with different
 * estimators may align against the same pyramids at the same time.  An unknown value or a NULL ctx ->
 * DVO_B200_ERR_INVALID_ARGUMENT (the setting is unchanged). */
int dvo_b200_set_estimator(dvo_b200_ctx* ctx, int32_t estimator);
/* the ctx's dvo_b200_estimator, or DVO_B200_ERR_INVALID_ARGUMENT for a NULL ctx */
int dvo_b200_get_estimator(const dvo_b200_ctx* ctx);

/* ---- image pyramid (replaces RgbdCameraPyramid::create + RgbdImagePyramid::build +
 *      RgbdImage::buildAccelerationStructure, rgbd_image.cpp:156-172,283-296,534-543) ---------- */
/* intensity/depth: HOST pointers to height*width float32, row-major; depth in metres, NaN = invalid
 * (what benchmark_slam.cpp:46-93 produces).  K = fx, fy, ox, oy of level 0.  levels >= 1.
 * Uploads, builds all levels (2x2 mean / subsample / central differences) and the default
 * point-selection masks on the device.  Asynchronous on the ctx stream; host buffers must stay
 * valid until dvo_b200_synchronize() unless they are not pinned (then the copy is staged). */
int dvo_b200_pyramid_create(dvo_b200_ctx* ctx, const float* intensity, const float* depth, int32_t width,
                            int32_t height, float fx, float fy, float ox, float oy, int32_t levels,
                            dvo_b200_pyramid** out);
/* n images with identical geometry; intensity/depth point to n consecutive images. */
int dvo_b200_pyramid_create_batch(dvo_b200_ctx* ctx, int32_t n, const float* intensity, const float* depth,
                                  int32_t width, int32_t height, float fx, float fy, float ox, float oy,
                                  int32_t levels, dvo_b200_pyramid** out /* n handles */);
/* N2 row (surface_pyramid.cpp:65-105, benchmark_slam.cpp:58-77): 8-bit grey + 16-bit raw depth in,
 * conversion (u16*scale, 0 -> NaN; u8 -> f32) fused into the upload. */
int dvo_b200_pyramid_create_raw(dvo_b200_ctx* ctx, const uint8_t* grey, const uint16_t* raw_depth, float depth_scale,
                                int32_t width, int32_t height, float fx, float fy, float ox, float oy,
                                int32_t levels, dvo_b200_pyramid** out);
/* n images with identical geometry; grey / raw_depth point to n consecutive images. */
int dvo_b200_pyramid_create_raw_batch(dvo_b200_ctx* ctx, int32_t n, const uint8_t* grey, const uint16_t* raw_depth,
                                      float depth_scale, int32_t width, int32_t height, float fx, float fy, float ox,
                                      float oy, int32_t levels, dvo_b200_pyramid** out /* n handles */);
/* 8-bit BGR (interleaved, the order cv::imread(file, 1) returns) + 16-bit raw depth in: cv::cvtColor(rgb, grey,
 * CV_BGR2GRAY) + convertTo(CV_32F) of the loader (benchmark_slam.cpp:50-68) and convertRawDepthImageSse run on the
 * device.  Grey = (1868 B + 9617 G + 4899 R + 8192) >> 14, OpenCV's 8-bit fixed-point BGR2GRAY. */
int dvo_b200_pyramid_create_bgr_batch(dvo_b200_ctx* ctx, int32_t n, const uint8_t* bgr, const uint16_t* raw_depth,
                                      float depth_scale, int32_t width, int32_t height, float fx, float fy, float ox,
                                      float oy, int32_t levels, dvo_b200_pyramid** out /* n handles */);
/* Input forms of dvo_b200_pyramid_create_masked_batch */
typedef enum dvo_b200_input_format {
  DVO_B200_INPUT_FLOAT32 = 0,        /* float intensity + float depth in metres (NaN = invalid), as dvo_b200_pyramid_create_batch */
  DVO_B200_INPUT_GREY8_DEPTH16 = 1,  /* 8-bit grey + 16-bit raw depth, as dvo_b200_pyramid_create_raw_batch */
  DVO_B200_INPUT_BGR8_DEPTH16 = 2    /* 8-bit interleaved BGR + 16-bit raw depth, as dvo_b200_pyramid_create_bgr_batch */
} dvo_b200_input_format;
/* The create calls above with a REFERENCE MASK per image: pixels the caller knows to be wrong (dynamic objects, the robot's
 * own body, specular or over-exposed areas, a vignetted border) never become constraints when the pyramid is the reference
 * of an alignment.  format: a dvo_b200_input_format (anything else -> DVO_B200_ERR_INVALID_ARGUMENT, nothing is created);
 * image / depth as in the call that format names; depth_scale is ignored for FLOAT32.  Host pointers are staged and may be
 * pageable or pinned, as in the other create calls.
 *   masks: n*height*width bytes, image i at i*height*width, row-major; nonzero = usable, 0 = excluded (an OpenCV CV_8U
 *     mask).  NULL: no mask, the pyramids are those of the call the format names, bit for bit.  An all-nonzero mask gives
 *     the same bits as no mask in every plane, selection and result.
 *   Coarser levels: a pixel of level l is usable iff every level-0 pixel of its footprint [x 2^l, (x+1) 2^l) x
 *     [y 2^l, (y+1) 2^l) is usable (an AND over each 2x2 block, level by level, the chain of the 2x2 intensity mean; the
 *     depth subsample point lies inside the footprint).
 *   Selection: at every level and for any thresholds, a pixel is selected iff isPointOk(ti, td) holds AND it is usable.
 *     Everything that follows from the selection follows the mask: LevelStats.valid_pixels (S), the odd last point
 *     (dropped by the reference estimator, re-admitted by the corrected one), dvo_b200_pyramid_select, the residual and
 *     intensity error images.  max_valid_pixels does not change.
 *   Reference role only: the mask does not change the pyramid as the CURRENT image of an alignment (its pixels stay valid
 *     bilinear taps) nor dvo_b200_pyramid_download.  dvo_b200_pyramid_create_masked_batch_roles with
 *     DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT makes the mask act in both roles.
 *   Fixed at creation: a pyramid's mask never changes, so sharing it across contexts and threads needs no new rule. */
int dvo_b200_pyramid_create_masked_batch(dvo_b200_ctx* ctx, int32_t n, int32_t format, const void* image, const void* depth,
                                         float depth_scale, const uint8_t* masks, int32_t width, int32_t height, float fx,
                                         float fy, float ox, float oy, int32_t levels, dvo_b200_pyramid** out /* n handles */);
/* Roles of a mask (bit set) */
#define DVO_B200_MASK_ROLE_REFERENCE 1   /* the selection: dvo_b200_pyramid_create_masked_batch */
#define DVO_B200_MASK_ROLE_CURRENT 2     /* the bilinear taps when the pyramid is the current image of an alignment */
/* dvo_b200_pyramid_create_masked_batch with a role set.  roles = DVO_B200_MASK_ROLE_REFERENCE: that call, bit for bit.
 * roles = DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT ("both"): the same pyramid as the reference of an
 * alignment (selection, S, odd last point, dvo_b200_pyramid_select unchanged), and as the CURRENT image a warped point is
 * rejected iff any of its four bilinear taps (u0, v0), (u0+1, v0), (u0, v0+1), (u0+1, v0+1) is unusable at that level, on
 * top of the bounds, NaN and occlusion tests -- the same rejection as a NaN depth at that tap.  The gradients of the usable
 * taps keep reading the true intensity and depth of unusable neighbours, so the ring of valid pixels next to an excluded
 * region stays.  Both stages of an iteration see the same points: n, P_k, the log-likelihood, A and b, and the test hooks
 * (dvo_b200_residual_image, dvo_b200_intensity_error_image, dvo_b200_linearize) follow, with both estimators.
 * dvo_b200_pyramid_download of such a pyramid returns Z = NaN at the unusable pixels of each level; the other planes are
 * those of the unmasked build.  Any other roles value -> DVO_B200_ERR_INVALID_ARGUMENT, nothing is created.
 * masks == NULL: the unmasked pyramids whatever the roles.  Fixed at creation, as the mask itself. */
int dvo_b200_pyramid_create_masked_batch_roles(dvo_b200_ctx* ctx, int32_t n, int32_t format, const void* image,
                                               const void* depth, float depth_scale, const uint8_t* masks, int32_t roles,
                                               int32_t width, int32_t height, float fx, float fy, float ox, float oy,
                                               int32_t levels, dvo_b200_pyramid** out /* n handles */);
/* One plane of a batch of images in DEVICE memory (dvo_b200_pyramid_create_device_batch): row y of image i starts at
 * (const char*)data + i * image_bytes + y * row_bytes, its pixels packed.  A cropped view of a larger image is a plane
 * whose data points at the crop's first pixel, with the larger image's row_bytes. */
typedef struct dvo_b200_device_plane {
  const void* data;     /* device (or managed) memory on the context's device, aligned to the element size */
  int64_t row_bytes;    /* >= width * bytes per pixel of the plane, a multiple of the element size */
  int64_t image_bytes;  /* image i starts at data + i * image_bytes; >= 0, a multiple of the element size (0: every image
                         * reads the same plane, e.g. one mask of the robot's body or a vignette for the whole batch) */
} dvo_b200_device_plane;
/* dvo_b200_pyramid_create_masked_batch_roles from planes already in device memory (frames decoded, rendered, rectified or
 * cropped on the GPU; masks from a segmentation network), without a host round trip: the same pyramids, bit for bit, as
 * that call with the same format, values, masks and roles -- every plane, the selection, S, the odd last point, the usable
 * bits and the current-role masking.
 *   Planes by format (element size, bytes per pixel): FLOAT32 image and depth (4, 4); GREY8_DEPTH16 grey (1, 1) and raw
 *     depth (2, 2); BGR8_DEPTH16 interleaved BGR (1, 3) and raw depth (2, 2); masks (1, 1), nonzero = usable, NULL: no mask
 *     (the unmasked pyramids of the format).  depth_scale is ignored for FLOAT32.
 *   Reads in place: depth and masks are read by the build's kernels where they lie (depth by every level's kernels); only
 *     BGR is reduced to 8-bit grey in the context's staging memory first.  Nothing is copied from the host:
 *     dvo_b200_h2d_bytes does not move.
 *   Stream order: all work is enqueued on dvo_b200_stream(ctx), and the call does not synchronise.  The inputs must be
 *     ready in that stream's order: make that stream wait for their producer (cudaStreamWaitEvent), or create the context
 *     on the producer's stream (dvo_b200_create(device, stream, ...)).  The caller must not modify or free the inputs until
 *     the work this call enqueued has completed (record an event on dvo_b200_stream(ctx) after the call and wait for it),
 *     as with the source of cudaMemcpyAsync.  The pyramids themselves follow the rules of every other pyramid.
 *   Validation (DVO_B200_ERR_INVALID_ARGUMENT with dvo_b200_last_error set, and nothing is created): a NULL
 *     image, depth or data pointer; an unknown format or role set (as dvo_b200_pyramid_create_masked_batch_roles); a
 *     row_bytes below width * bytes per pixel or not a multiple of the element size; a negative image_bytes or one that is
 *     not a multiple of the element size; a data pointer not aligned to the element size; and a first or last byte of a
 *     plane's extent that cudaPointerGetAttributes does not report as device or managed memory of the context's device --
 *     pageable or pinned host memory is refused, never copied. */
int dvo_b200_pyramid_create_device_batch(dvo_b200_ctx* ctx, int32_t n, int32_t format, const dvo_b200_device_plane* image,
                                         const dvo_b200_device_plane* depth, float depth_scale,
                                         const dvo_b200_device_plane* masks /* NULL: no mask */, int32_t roles, int32_t width,
                                         int32_t height, float fx, float fy, float ox, float oy, int32_t levels,
                                         dvo_b200_pyramid** out /* n handles */);
/* ---- distorted cameras: undistortion through a remap in the pyramid build -------------------------------------------
 * The tracker projects with a pinhole K.  Frames of a real lens are first remapped to a pinhole camera K_new: output pixel
 * (x, y) of a rectified frame reads the input frame at (sx, sy) = (map_x[y*w + x], map_y[y*w + x]).
 *
 * dvo_b200_undistort_map: the map of OpenCV's plumb-bob model with R = I, as cv::initUndistortRectifyMap(K, dist, I, K_new,
 * (width, height), CV_32FC1) computes it.  Host only: no context, no GPU.  K and K_new are fx, fy, cx, cy; dist is k1, k2,
 * p1, p2, k3.  For each output pixel (u, v), in double precision and in this order (a*b+c means (a*b)+c, no fused
 * multiply-add):
 *   x  = (u - cx') / fx'                       y  = (v - cy') / fy'            (K_new = fx', fy', cx', cy')
 *   r2 = x*x + y*y
 *   kr = ((k3*r2 + k2)*r2 + k1)*r2                                             (the radial factor minus 1)
 *   dx = x*kr + ((2*p1)*x*y + p2*(r2 + 2*x*x))  dy = y*kr + (p1*(r2 + 2*y*y) + (2*p2)*x*y)
 *   map_x = (cx + (fx/fx')*(u - cx')) + fx*dx  map_y = (cy + (fy/fy')*(v - cy')) + fy*dy
 * then each map value is rounded once to float.  This is fx*(x*(1 + kr) + tangential) + cx, the plumb-bob model, written
 * so that zero coefficients with K_new = K give exact integer coordinates (dx = 0 and cx + (u - cx) = u).  width*height
 * floats per map.  A NULL pointer, a non-positive size or a non-finite K, K_new or dist -> DVO_B200_ERR_INVALID_ARGUMENT. */
int dvo_b200_undistort_map(int32_t width, int32_t height, const double K[4], const double dist[5], const double K_new[4],
                           float* map_x, float* map_y);
/* A rectifier: one map, uploaded once to the context's device, through which later create calls remap their frames.  Any
 * camera model works through its map (fisheye maps or stereo rectification from OpenCV, say).
 *   in_width x in_height: the frames the create calls take (>= 2 x 2).  width x height: the rectified frames, i.e. level 0 of
 *     the pyramids; map_x / map_y: HOST arrays of width*height floats, input pixel coordinates (pixel centres at integers,
 *     OpenCV's convention).  K_new: fx, fy, cx, cy of the rectified camera, level 0's intrinsics.  Copied: the caller's
 *     arrays may be freed when the call returns.  Synchronises.  dvo_b200_h2d_bytes grows by the 8*width*height bytes of
 *     the map, once.
 *   A rectifier belongs to its context: only create calls on that context take it.  dvo_b200_rectifier_release may be
 *   called as soon as the create calls that used it have returned, with their work still queued; its memory is freed in
 *   the context's stream order after that work, with no host synchronisation.  Release every rectifier of a context before
 *   destroying the context. */
typedef struct dvo_b200_rectifier dvo_b200_rectifier;
int dvo_b200_rectifier_create(dvo_b200_ctx* ctx, int32_t in_width, int32_t in_height, int32_t width, int32_t height,
                              const float* map_x, const float* map_y, const float K_new[4], dvo_b200_rectifier** out);
int dvo_b200_rectifier_release(dvo_b200_rectifier* r);
/* Rectified creates: the frames (in_width x in_height, given as width / height, which must equal the rectifier's) are
 * remapped into the context's staging memory, then built exactly as dvo_b200_pyramid_create_masked_batch_roles builds
 * FLOAT32 frames of the rectifier's width x height with intrinsics K_new.  format, masks (nonzero = usable, in the INPUT
 * geometry), roles, depth_scale and levels as in that call.
 *   For output pixel (x, y) with (sx, sy) = map(x, y), in float32:
 *     valid iff 0 <= sx <= in_width - 1 and 0 <= sy <= in_height - 1 (a NaN or infinite coordinate is invalid);
 *     taps x0 = min(floor(sx), in_width - 2), ax = sx - x0, y0 = min(floor(sy), in_height - 2), ay = sy - y0;
 *     intensity = bilinear, each operation rounded to nearest, no contraction:
 *       top = (1-ax)*I(x0,y0) + ax*I(x0+1,y0), bot = (1-ax)*I(x0,y0+1) + ax*I(x0+1,y0+1), I = (1-ay)*top + ay*bot
 *       from 8-bit grey or float32; BGR is first reduced to 8-bit grey exactly as dvo_b200_pyramid_create_bgr_batch does;
 *     depth = the nearest tap, never blended (a blend across a depth edge invents a surface): Z(x0 + (ax >= 0.5),
 *       y0 + (ay >= 0.5)), float32 metres as given or u16 * depth_scale with 0 -> NaN, as the raw create calls convert;
 *     an invalid pixel gets I = NaN and Z = NaN: it is never a point or a tap, and the 2x2 mean carries the NaN into every
 *       coarse pixel whose footprint touches the area without source (a zero would be a false intensity there);
 *     mask: usable iff the pixel is valid and its four intensity taps are usable.
 *   The pyramids equal, bit for bit, those of dvo_b200_pyramid_create_masked_batch_roles(FLOAT32) on the rectified planes
 *   and mask (masks == NULL: no mask, whatever the roles), with the rectifier's size and K_new.
 * dvo_b200_pyramid_create_rectified_batch: HOST pointers to n frames, staged like dvo_b200_pyramid_create_masked_batch_roles
 *   (dvo_b200_h2d_bytes grows by the input bytes only).
 * dvo_b200_pyramid_create_rectified_device_batch: dvo_b200_device_plane inputs, validated and ordered exactly as in
 *   dvo_b200_pyramid_create_device_batch; nothing is copied from the host.
 * A NULL ctx or rectifier, a rectifier of another context, a width / height other than the rectifier's input size, or any
 * argument the corresponding unrectified call refuses -> DVO_B200_ERR_INVALID_ARGUMENT, and nothing is created. */
int dvo_b200_pyramid_create_rectified_batch(dvo_b200_ctx* ctx, const dvo_b200_rectifier* rect, int32_t n, int32_t format,
                                            const void* image, const void* depth, float depth_scale, const uint8_t* masks,
                                            int32_t roles, int32_t width, int32_t height, int32_t levels,
                                            dvo_b200_pyramid** out /* n handles */);
int dvo_b200_pyramid_create_rectified_device_batch(dvo_b200_ctx* ctx, const dvo_b200_rectifier* rect, int32_t n, int32_t format,
                                                   const dvo_b200_device_plane* image, const dvo_b200_device_plane* depth,
                                                   float depth_scale, const dvo_b200_device_plane* masks /* NULL: no mask */,
                                                   int32_t roles, int32_t width, int32_t height, int32_t levels,
                                                   dvo_b200_pyramid** out /* n handles */);
/* ---- unregistered depth: a separate depth camera reprojected into the colour camera in the pyramid build --------------
 * The tracker needs every pixel's depth measured along the ray of its intensity.  A sensor whose depth comes from its own
 * camera (time of flight, a stereo pair) some centimetres from the colour camera first has its depth registered: every depth
 * pixel is moved into the colour camera, whose geometry the pyramids keep.
 *
 * dvo_b200_depth_rays: the ray tables of a depth camera of dw x dh pixels, in normalised coordinates (z = 1), rounded once
 * to float.  Host only: no context, no GPU.  K_depth = fx, fy, cx, cy.  cx_ray / cy_ray [dh][dw]: the ray through pixel
 * centre (u, v); kx_ray / ky_ray [dh+1][dw+1]: the ray through pixel corner (u - 0.5, v - 0.5), u in 0..dw, v in 0..dh.
 *   dist == NULL (pinhole): x = (u - cx) / fx, y = (v - cy) / fy in double.
 *   dist = k1, k2, p1, p2, k3 (OpenCV's plumb-bob model): the pixel's distorted coordinates xd = (u - cx) / fx,
 *     yd = (v - cy) / fy are undistorted by Newton's method in double, from (x, y) = (xd, yd), per point, in this order (a*b+c
 *     means (a*b)+c, products left to right, no fused multiply-add):
 *       r2 = x*x + y*y;  R = 1 + ((k3*r2 + k2)*r2 + k1)*r2;  dR = k1 + (2*k2 + 3*k3*r2)*r2
 *       ex = x*R + 2*p1*x*y + p2*(r2 + 2*x*x) - xd;  ey = y*R + p1*(r2 + 2*y*y) + 2*p2*x*y - yd
 *       stop when |ex| < 1e-12 and |ey| < 1e-12; otherwise, after DVO_B200_DEPTH_RAYS_MAX_ITER updates, fail;
 *       a = R + 2*x*x*dR + 2*p1*y + 6*p2*x;  b = 2*x*y*dR + 2*p1*x + 2*p2*y;  d = R + 2*y*y*dR + 6*p1*y + 2*p2*x
 *       det = a*d - b*b;  x' = x - (d*ex - b*ey) / det;  y' = y - (a*ey - b*ex) / det
 *   A NULL table or K_depth, dw or dh < 2, a non-finite K_depth or dist, fx or fy <= 0, or a point that does not converge
 *   -> DVO_B200_ERR_INVALID_ARGUMENT (the tables are then undefined). */
#define DVO_B200_DEPTH_RAYS_MAX_ITER 100
int dvo_b200_depth_rays(int32_t dw, int32_t dh, const double K_depth[4], const double dist[5] /* NULL: pinhole */, float* cx_ray,
                        float* cy_ray, float* kx_ray, float* ky_ray);
/* A depth registration: a depth camera given by its ray tables (any camera model works through them, as any remap works
 * through a rectifier's map), the rigid transform T_color_depth (row-major 4x4 double, p_color = T * p_depth, metres) and the
 * target pinhole colour camera of width x height pixels and intrinsics K = fx, fy, cx, cy (level 0 of the pyramids).
 *   The tables are HOST arrays as dvo_b200_depth_rays writes them; they are uploaded once to the context's device and the
 *   call synchronises, so the caller's arrays may be freed when it returns.  dvo_b200_h2d_bytes grows by their
 *   4 * (2*dw*dh + 2*(dw+1)*(dh+1)) bytes, once.  T is stored as float R (9 values) and t (3 values), each rounded once.
 *   Refused with DVO_B200_ERR_INVALID_ARGUMENT: a NULL pointer, dw or dh < 2, a non-positive width or height, a non-finite
 *   ray, T or K, fx or fy <= 0, a bottom row of T other than (0, 0, 0, 1), max|R^T R - I| > 1e-6 or det R <= 0.
 *   A registration belongs to its context, and dvo_b200_depth_registration_release frees it in the context's stream order
 *   with no host synchronisation, exactly as dvo_b200_rectifier_release does.  Release every registration of a context
 *   before destroying the context. */
typedef struct dvo_b200_depth_registration dvo_b200_depth_registration;
int dvo_b200_depth_registration_create(dvo_b200_ctx* ctx, int32_t dw, int32_t dh, const float* cx_ray, const float* cy_ray,
                                       const float* kx_ray, const float* ky_ray, const double T_color_depth[16], int32_t width,
                                       int32_t height, const float K[4], dvo_b200_depth_registration** out);
int dvo_b200_depth_registration_release(dvo_b200_depth_registration* reg);
/* Registered creates.  In float32, every operation rounded to nearest (no fused multiply-add), for each depth pixel (u, v)
 * of image i:
 *   d: float32 metres as given, or u16 * depth_scale with 0 -> NaN as the raw creates convert; skipped unless d is finite
 *     and d > 0.
 *   For a ray (rx, ry): P = (rx*d, ry*d, d), Pc = R*P + t with each component ((r0*X + r1*Y) + r2*Z) + t.
 *   The value is Zc of the centre ray; skipped unless Zc > 0.
 *   Footprint: the four corner rays of the pixel project to x = fx*(Xc/Zc) + cx, y = fy*(Yc/Zc) + cy (divide, multiply,
 *     add).  Skipped unless all four corners have Zc > 0 and every |x|, |y| < 2^20.  It covers the colour columns
 *     ceil(xmin) .. ceil(xmax) - 1 and rows ceil(ymin) .. ceil(ymax) - 1 (half-open, so neighbours on a continuous surface
 *     tile without cracks); skipped if either extent exceeds DVO_B200_REGISTRATION_MAX_FOOTPRINT; then clipped to the image.
 *   Depth test: each colour pixel keeps the minimum Zc of the depth pixels that cover it, whatever their order.  A colour
 *     pixel nothing covers gets NaN depth: it is never a point or a tap (the part of the scene the colour camera sees and
 *     the depth camera does not).
 * Intensity and masks (nonzero = usable) stay in the colour geometry:
 *   rect == NULL: the colour frames are width x height = the registration's target size; the intensity is used as given
 *     (float32, 8-bit grey converted exactly, BGR reduced as dvo_b200_pyramid_create_bgr_batch reduces it).
 *   rect != NULL (a distorted colour camera): its output size and K_new equal the registration's target, width x height is
 *     its input size, and intensity and masks go through its map with the rules of the rectified creates.  Depth comes from
 *     the registration, never from the map.
 * The pyramids equal, bit for bit, those of dvo_b200_pyramid_create_masked_batch_roles(FLOAT32) on the registered
 * intensity and depth planes (and mask), with the registration's width x height and K.  With the identity registration
 * (the same size, the pinhole rays of K, T = I) every colour pixel is covered by its own depth pixel alone and Zc = d, so
 * the pyramids are those of the unregistered create of the same format.
 * dvo_b200_pyramid_create_registered_batch: HOST pointers to n colour frames of width x height and n depth frames of the
 *   registration's dw x dh, staged like dvo_b200_pyramid_create_masked_batch_roles (dvo_b200_h2d_bytes grows by the input
 *   bytes only).
 * dvo_b200_pyramid_create_registered_device_batch: dvo_b200_device_plane inputs, validated and ordered exactly as in
 *   dvo_b200_pyramid_create_device_batch, the depth plane against dw x dh; nothing is copied from the host.
 * A NULL ctx or registration, a registration or rectifier of another context, a colour size other than the target (or the
 * rectifier's input size), a rectifier whose output size or K_new differs from the target, or any argument the
 * corresponding unregistered call refuses -> DVO_B200_ERR_INVALID_ARGUMENT, and nothing is created. */
#define DVO_B200_REGISTRATION_MAX_FOOTPRINT 8
int dvo_b200_pyramid_create_registered_batch(dvo_b200_ctx* ctx, const dvo_b200_depth_registration* reg,
                                             const dvo_b200_rectifier* rect /* NULL: pinhole colour camera */, int32_t n,
                                             int32_t format, const void* image, const void* depth, float depth_scale,
                                             const uint8_t* masks, int32_t roles, int32_t width, int32_t height, int32_t levels,
                                             dvo_b200_pyramid** out /* n handles */);
int dvo_b200_pyramid_create_registered_device_batch(dvo_b200_ctx* ctx, const dvo_b200_depth_registration* reg,
                                                    const dvo_b200_rectifier* rect /* NULL: pinhole colour camera */, int32_t n,
                                                    int32_t format, const dvo_b200_device_plane* image,
                                                    const dvo_b200_device_plane* depth, float depth_scale,
                                                    const dvo_b200_device_plane* masks /* NULL: no mask */, int32_t roles,
                                                    int32_t width, int32_t height, int32_t levels,
                                                    dvo_b200_pyramid** out /* n handles */);
/* Role set a pyramid was created with: 0 (no mask), DVO_B200_MASK_ROLE_REFERENCE, or
 * DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT; DVO_B200_ERR_INVALID_ARGUMENT for a null handle. */
int dvo_b200_pyramid_mask_roles(const dvo_b200_pyramid* p);
int dvo_b200_pyramid_device(const dvo_b200_pyramid* p);   /* CUDA ordinal the pyramid lives on (-1: null handle) */
int dvo_b200_pyramid_retain(dvo_b200_pyramid* p);   /* boost::shared_ptr semantics of RgbdImagePyramidPtr */
/* Any context may use a pyramid, also while its build is still queued on the building context's stream: every call
 * waits for the build on the device.  A pyramid may be released from any host thread as soon as the calls that used it
 * have returned, on any context, including dvo_b200_match_batch_device with its work still queued: its memory is only
 * rebuilt after that work.  Does not change the calling thread's current device. */
int dvo_b200_pyramid_release(dvo_b200_pyramid* p);
int dvo_b200_pyramid_num_levels(const dvo_b200_pyramid* p);
int dvo_b200_pyramid_level_info(const dvo_b200_pyramid* p, int32_t level, int32_t* width, int32_t* height, float K[4]);
/* Debug/test read-back of one level: 6 planes (I, Z, Ix, Iy, Zx, Zy) of h*w floats into host memory.
 * Z is the tracker's masked depth: NaN wherever the reference would reject the pixel as a bilinear
 * tap or as a reference point (any of I,Z,Ix,Iy,Zx,Zy NaN).  Synchronises.  ctx may be NULL: pyramids are shared objects
 * that can outlive the context that built them (boost::shared_ptr<RgbdImagePyramid>); the read then waits for the
 * pyramid's own build to finish and uses no context at all.  Does not change the calling thread's current device. */
int dvo_b200_pyramid_download(dvo_b200_ctx* ctx, const dvo_b200_pyramid* p, int32_t level, float* planes6);
/* PointSelection::select result (point_selection.cpp:89-152) for the given thresholds: number of
 * selected points S and (optional) h*w byte mask.  Synchronises. */
int dvo_b200_pyramid_select(dvo_b200_ctx* ctx, dvo_b200_pyramid* p, int32_t level, float intensity_threshold,
                            float depth_threshold, int64_t* count, uint8_t* mask);

/* ---- alignment ---------------------------------------------------------------------------- */
/* DenseTracker::match(RgbdImagePyramid& reference, RgbdImagePyramid& current, Result&)
 * (dense_tracking.cpp:123-129).  T_init: row-major 4x4 Result.Transformation on entry (read iff
 * cfg->use_initial_estimate), may be NULL.  Blocks until the result is on the host. */
int dvo_b200_match(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                   dvo_b200_pyramid* current, const double* T_init, dvo_b200_result* result);
/* n independent alignments (the TBB fan-outs of local_tracker.cpp:180-184 and
 * keyframe_graph.cpp:587-590 as one call).  T_init: n*16 doubles or NULL.  iteration_stats: optional
 * n*max_iteration_stats entries, pair p's iterations start at p*max_iteration_stats, in order. */
int dvo_b200_match_batch(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                         dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents,
                         const double* T_init, dvo_b200_result* results,
                         dvo_b200_iteration_stats* iteration_stats, int32_t max_iteration_stats);
/* Asynchronous variant: enqueues the batch and leaves the n results in DEVICE memory
 * (d_results: device pointer to n dvo_b200_result) so they can be gathered with NCCL without a
 * host round trip.  No synchronisation. */
int dvo_b200_match_batch_device(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                                dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents,
                                const double* T_init, void* d_results);

/* ---- one process, several GPUs (SURVEY.md 8e) ----------------------------------------------------
 * The reference's batch producers are single-process C++ loops over independent match() calls
 * (constraint_proposal_validator.cpp:141-146, keyframe_graph.cpp:587-590).  A dvo_b200_sharded owns one context per
 * device; a batch of n pairs is cut into contiguous shards of pair indices (dvo_b200_shard_range: the remainder goes to
 * the first shards -- the same partition the multi-process path dvo_slam_b200/distributed.py uses), each shard runs on
 * its own host thread and device, and every shard writes its results into its range of the caller's host array.  The
 * alignments exchange nothing, so a one-process caller needs no communicator; across processes the gather is one NCCL
 * all-gather of the records left in device memory by dvo_b200_match_batch_device. */
typedef struct dvo_b200_sharded dvo_b200_sharded;
/* devices: n_devices CUDA ordinals, or NULL for 0..n_devices-1 (an ordinal may repeat: two shards on one GPU). */
int dvo_b200_sharded_create(int32_t n_devices, const int32_t* devices, dvo_b200_sharded** out);
int dvo_b200_sharded_destroy(dvo_b200_sharded* s);
int32_t dvo_b200_sharded_num_shards(const dvo_b200_sharded* s);
dvo_b200_ctx* dvo_b200_sharded_ctx(dvo_b200_sharded* s, int32_t shard);     /* the shard's context (owned by s) */
const char* dvo_b200_sharded_last_error(dvo_b200_sharded* s);
int dvo_b200_shard_range(int64_t total, int32_t n_shards, int32_t shard, int64_t* begin, int64_t* end);
/* n images -> n pyramids, image i on the device of the shard that owns index i of n; blocks until the uploads are done */
int dvo_b200_sharded_pyramid_create_batch(dvo_b200_sharded* s, int32_t n, const float* intensity, const float* depth,
                                          int32_t width, int32_t height, float fx, float fy, float ox, float oy,
                                          int32_t levels, dvo_b200_pyramid** out /* n handles */);
int dvo_b200_sharded_pyramid_create_raw_batch(dvo_b200_sharded* s, int32_t n, const uint8_t* grey, const uint16_t* raw_depth,
                                              float depth_scale, int32_t width, int32_t height, float fx, float fy,
                                              float ox, float oy, int32_t levels, dvo_b200_pyramid** out);
/* dvo_b200_match_batch over all shards: pair i must live on the device of the shard that owns index i of n (as the two
 * calls above place them), else DVO_B200_ERR_INVALID_ARGUMENT.  Same result layout as dvo_b200_match_batch. */
int dvo_b200_match_batch_sharded(dvo_b200_sharded* s, const dvo_b200_config* cfg, int32_t n,
                                 dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents,
                                 const double* T_init, dvo_b200_result* results,
                                 dvo_b200_iteration_stats* iteration_stats, int32_t max_iteration_stats);

/* One evaluation of the residual stage at a fixed transform (test / debug; also the basis of
 * DenseTracker::computeIntensityErrorImage, dense_tracking.cpp:378-444): 7 planes
 * {e.i, e.z, e.idx, e.idy, e.zdx, e.zdy, z_ref} of h*w floats, NaN where invalid.  T: row-major
 * 4x4 double "estimate" (reference -> current).  Returns n (valid constraints) in *count. */
int dvo_b200_residual_image(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                            dvo_b200_pyramid* current, int32_t level, const double* T, float* planes7,
                            int64_t* count);
/* DenseTracker::computeIntensityErrorImage (dense_tracking.cpp:378-444): image = h*w floats on the host,
 * |intensity residual| at every selected reference pixel whose warped residual is valid, 0 elsewhere (the odd
 * last selected point included: the reference's SSE residual loop never visits it; with DVO_B200_ESTIMATOR_CORRECTED it
 * is a constraint like any other and appears here and in dvo_b200_residual_image).  T as above; the selection
 * thresholds come from cfg.  *count (optional) = residuals written. */
int dvo_b200_intensity_error_image(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                                   dvo_b200_pyramid* current, int32_t level, const double* T, float* image,
                                   int64_t* count);
/* One linearisation at a fixed transform (test hook mirroring dense_tracking.cpp:271-343):
 * use_weights=0 -> w=1 (first iteration on a level), else Student-t weights from prev_precision. */
int dvo_b200_linearize(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                       dvo_b200_pyramid* current, int32_t level, const double* T, int32_t use_weights,
                       const float* prev_precision, int64_t* count, float* precision_out, float* ll_out,
                       double* A_out, double* b_out);

/* ---- photometric mode: an affine brightness change per pair, estimated jointly with the pose ----------------------
 * Auto exposure and white balance change the intensity of consecutive frames by a global gain and offset, which the
 * brightness-constancy residual cannot absorb.  In this mode every alignment estimates 8 unknowns, the pose xi, a gain
 * alpha and a bias beta, with the model I_cur(w(x)) ~ alpha I_ref(x) + beta (intensities on the 0..255 scale of the
 * pyramid).  With either estimator and with current-role masks; the default entry points are unchanged.  Operation by
 * operation:
 *   residual   e_i = c_i I_cur(w) - c_i fmaf(alpha, I_ref, beta), c_i = 1/255, with (alpha, beta) rounded to float: at
 *              (1, 0) it is the default e_i bit for bit.  The depth residual, the validity of a point, the occlusion test
 *              and the selection do not depend on (alpha, beta).
 *   weights, scale, log-likelihood: the estimator's own formulas over the new e_i (REFERENCE: with its three quirks).
 *   normal equations: 8 x 8 over (xi, alpha, beta) with W = w P_k.  The intensity row adds de_i/dalpha = -c_i I_ref and
 *              de_i/dbeta = -c_i; the depth row has zeros there.  Jacobians at the untransformed point, as by default.
 *   prior      mu acts on the pose block as by default (A_ii += mu, b_i += mu log(initial)_i for i < 6); none on alpha, beta.
 *   solve      8 x 8 LDL^T in fp64 with the pivot rule of the 6 x 6.  The pose is updated as by default, alpha += dalpha,
 *              beta += dbeta (fp64), with the pose: an increment is applied when the pose's is, and a rejected iteration
 *              (LogLikelihoodDecreased, TooFewConstraints) reverts all 8 together.
 *   termination IncrementTooSmall tests the 6 pose components only; precision keeps its meaning.  The rest is unchanged.
 *   levels     (alpha, beta) carry over from level to level unchanged (the 2 x 2 mean commutes with an affine map).
 *   outputs    transformation and log_likelihood keep their meaning.  information is the Schur complement of the 8 x 8
 *              (prior included) onto the pose, A_xx - A_xp A_pp^-1 A_px, times 0.008^2 as by default; iteration stats carry
 *              the pose part of the increment and the same Schur complement; level stats are unchanged.
 * Outputs in device memory and several GPUs: dvo_b200_match_batch_modes_device and _modes_sharded below. */

/* dvo_b200_match_batch in the photometric mode.  photometric_init: 2n doubles (alpha, beta) per pair, or NULL = (1, 0) each;
 * photometric: 2n doubles out, the final (alpha, beta) of each pair.  A NULL photometric or a non-finite photometric_init is
 * refused with DVO_B200_ERR_INVALID_ARGUMENT before anything is uploaded or launched; every other argument is checked as
 * dvo_b200_match_batch checks it. */
int dvo_b200_match_batch_photometric(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                                     dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents,
                                     const double* T_init, const double* photometric_init, dvo_b200_result* results,
                                     double* photometric, dvo_b200_iteration_stats* iteration_stats,
                                     int32_t max_iteration_stats);
/* The test hooks at a fixed (alpha, beta) = ab (finite, else DVO_B200_ERR_INVALID_ARGUMENT), on the same kernel instance as
 * the photometric match.  dvo_b200_linearize_photometric returns the whole 8 x 8 A (row-major, no prior) and the 8 of b. */
int dvo_b200_residual_image_photometric(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                                        dvo_b200_pyramid* current, int32_t level, const double* T, const double ab[2],
                                        float* planes7, int64_t* count);
int dvo_b200_linearize_photometric(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                                   dvo_b200_pyramid* current, int32_t level, const double* T, const double ab[2],
                                   int32_t use_weights, const float* prev_precision, int64_t* count, float* precision_out,
                                   float* ll_out, double A_out[64], double b_out[8]);

/* ---- motion prior: a full 6 x 6 prior information per pair on the pose, in place of mu I -----------------------------
 * What a caller knows about the motion -- a constant-velocity prediction with the previous alignment's information, an
 * IMU or wheel-odometry preintegration with its covariance, the relative pose of a keyframe-graph edge -- enters each
 * alignment as a symmetric positive semi-definite Lambda_p (row-major, fp64), one per pair.  Definitions:
 *   T0       the initial estimate as the kernel reads it: T_init of the pair when cfg->use_initial_estimate is set and T_init
 *            is given, else the identity.
 *   initial  the reference's Revertable "initial" (dense_tracking.cpp:147-149, 259-261), T0 estimate^-1 at every iteration.
 *   li       log(initial) in the twist order of the engine, [v; omega].
 * Where the default path uses mu, this one uses Lambda_p:
 *   normal equations         A + Lambda_p          (default A + mu I)
 *   right-hand side          b + Lambda_p li       (default b + mu li)
 *   prior log-likelihood     li^T Lambda_p li      (default mu sum li^2)
 *   iteration information    A + Lambda_p          (default A + mu I)
 *   result information       (A_last + Lambda_p) 0.008^2
 * Result.log_likelihood keeps its meaning, with this prior term.  The accept test ignores the prior, as by default
 * (SURVEY Q18); termination, the Revertable handling and the levels are unchanged.  In the photometric mode Lambda_p acts on
 * the pose block of the 8 x 8 system, exactly where mu does (A_ij, b_i for i, j < 6, and the system whose Schur complement
 * is the information); there is no prior on (alpha, beta).
 * Units and coordinates: Lambda has the units of A, not of Result.information.  The prior is on eps where
 * estimate = exp(eps) T0; equivalently Result.transformation = T0^-1 exp(-eps), a right perturbation of the returned
 * transformation.  An IMU covariance Sigma in those coordinates gives Lambda = Sigma^-1; a previous alignment of the same
 * motion gives Lambda = Result.information / 0.008^2, because its A is in the same coordinates.
 * Arithmetic: b_i + sum_j Lambda_ij li_j is an in-order FMA chain over j and A_ij + Lambda_ij one addition, so Lambda = mu I
 * returns the bits of dvo_b200_match_batch[_photometric] with cfg->mu = mu in everything but the prior log-likelihood (and
 * with it log_likelihood), which may differ in the last bits; Lambda = 0 returns the bits of mu = 0 in everything.
 * Outputs in device memory and several GPUs: dvo_b200_match_batch_modes_device and _modes_sharded below. */

/* dvo_b200_match_batch with a prior information per pair.  prior_information: n * 36 doubles, pair p's Lambda at p * 36.
 * photometric NULL: the default 6-unknown mode; non-NULL: the photometric mode, photometric_init and photometric as in
 * dvo_b200_match_batch_photometric.  Refused with DVO_B200_ERR_INVALID_ARGUMENT before anything is staged, uploaded or
 * launched: a NULL prior_information; photometric_init without photometric; cfg->mu != 0 (the prior replaces mu I rather
 * than adding to it); a Lambda_p with a non-finite entry, with Lambda_ij != Lambda_ji (exact comparison) or with an
 * eigenvalue below -1e-9 max(1, max |Lambda_ij|); and everything dvo_b200_match_batch[_photometric] refuses.  A zero row
 * means no prior in that direction. */
int dvo_b200_match_batch_prior(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                               dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents,
                               const double* T_init, const double* prior_information, const double* photometric_init,
                               double* photometric, dvo_b200_result* results, dvo_b200_iteration_stats* iteration_stats,
                               int32_t max_iteration_stats);

/* ---- weight maps: each alignment's per-pixel Student-t weights and residuals at its returned pose, and an outlier mask --
 * The estimator down-weights every constraint by w = 7 / (5 + r^T P r); at convergence the pixels of a moving object, a
 * specularity or a depth edge are the ones with small w.  dvo_b200_match_batch_maps runs an alignment exactly as the
 * entry point without maps would, then one more kernel that writes these maps for every pair.  Definitions, with
 * L = cfg->last_level:
 *   kept iteration  the last iteration on level L whose pose was not reverted.  It supplies T^ (the estimate that
 *              Result.transformation inverts: T^ = Result.transformation^-1 up to rounding), P^ (the precision that
 *              iteration estimated, which is the iteration log's tdist_precision of that entry), n^ (its constraint
 *              count, levels[L].last_increment_valid_constraints) and, in the photometric mode, (alpha, beta) as returned.
 *   K T        K_cur,L * float(T^)[0:3, :] in float, in the operation order of the level kernel (the current image's
 *              level-L intrinsics).
 *   residuals  the residual record of every reference pixel of level L at K T, with the projection, bilinear blend,
 *              NaN test and occlusion test of the level kernel, and the current-role mask rejection where the current
 *              pyramid has one: residual_i = c_i I_cur(w) - c_i I_ref (photometric mode: c_i fmaf(alpha, I_ref, beta) with
 *              alpha, beta rounded to float), residual_z = Z_cur(w) - Z'(x).  Bit for bit planes 0 and 1 of
 *              dvo_b200_residual_image[_photometric] at the 4 x 4 se3 matrix of T^ (and (alpha, beta)).
 *   weight     w = 7 rcp(5 + d), d = r^T P^ r, with the operation sequence of the level kernel (rcp.approx: within a few
 *              ulp of 7 / (5 + d) in fp64).
 *   not a constraint   a pixel that is not selected, or is out of bounds, NaN or occluded at T^: NaN in all three
 *              maps.  With DVO_B200_ESTIMATOR_REFERENCE the odd last selected point is not a constraint either; with
 *              DVO_B200_ESTIMATOR_CORRECTED it is.  So exactly n^ weights are finite.
 *   NaN result a pair whose Result has NaN information (no accepted iteration on level L, or TooFewConstraints) gets NaN
 *              maps, a NaN P^ and an all-1 mask; its estimate is still written.
 *   mask       one byte per level-0 pixel of the reference: 0 iff its level-L parent (x >> L, y >> L) is a constraint with
 *              w < mask_weight, 1 otherwise (level-0 pixels without a parent, past an odd size, are 1).  It is the masks
 *              plane dvo_b200_pyramid_create_device_batch takes (nonzero = usable), so the outliers of one alignment can
 *              be kept out of the next alignment against the same keyframe without a host round trip.  No dilation.
 * Outputs, per requested plane: pair p's map starts at data + p * image_bytes, row y at + y * row_bytes.  The weight and
 * residual planes are float32 of level L's size, the mask uint8 of level 0's size. */
#define DVO_B200_MAPS_DEVICE 0   /* every pointer of the dvo_b200_weight_maps is device or managed memory of the ctx's device */
#define DVO_B200_MAPS_HOST 1     /* every pointer is host memory (pageable or pinned); the maps are copied back */
typedef struct dvo_b200_map_plane {
  void* data;            /* NULL: not written */
  int64_t row_bytes;     /* >= width * element size, a multiple of the element size */
  int64_t image_bytes;   /* >= height * row_bytes, a multiple of the element size */
} dvo_b200_map_plane;
typedef struct dvo_b200_weight_maps {
  int32_t memory;                 /* DVO_B200_MAPS_DEVICE or DVO_B200_MAPS_HOST: where every pointer below lies */
  dvo_b200_map_plane weight;      /* float32, level-L size of pair p's reference */
  dvo_b200_map_plane residual_i;  /* float32, residual_i */
  dvo_b200_map_plane residual_z;  /* float32, residual_z */
  dvo_b200_map_plane mask;        /* uint8, level-0 size */
  float mask_weight;              /* finite and > 0; read iff mask.data */
  double* estimate;               /* n * 16, the se3 matrix of T^ row-major (reference -> current), or NULL */
  float* precision;               /* n * 4, P^ row-major, or NULL */
} dvo_b200_weight_maps;

/* An alignment and its weight maps.  The arguments before maps are those of dvo_b200_match_batch_prior, with
 * prior_information NULL for the plain cfg->mu path and photometric NULL for the 6-unknown mode; results, photometric and
 * the iteration statistics are bit for bit those of dvo_b200_match_batch, _photometric or _prior with the same arguments,
 * for every estimator, current-role mask and launch plan.  One kernel launch more than that call (k_weight_maps, which
 * writes the mask in the same pass).  Synchronises as dvo_b200_match_batch does; with DVO_B200_MAPS_HOST the maps have been
 * copied back when it returns.  Refused with DVO_B200_ERR_INVALID_ARGUMENT before anything is staged, uploaded or launched:
 * a NULL maps; an unknown memory; no output requested; a row_bytes below the largest width of the batch times the element
 * size or not a multiple of it; an image_bytes below the largest height times row_bytes or not a multiple of the element
 * size; a misaligned pointer; under DVO_B200_MAPS_DEVICE a first or last byte of an output that cudaPointerGetAttributes
 * does not report as device or managed memory of the ctx's device, and under DVO_B200_MAPS_HOST one in device memory; a
 * non-finite or non-positive mask_weight with a mask; and everything the matching entry point refuses (a batch of mixed
 * sizes included: DVO_B200_ERR_SHAPE_MISMATCH). */
int dvo_b200_match_batch_maps(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                              dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents,
                              const double* T_init, const double* prior_information, const double* photometric_init,
                              double* photometric, dvo_b200_result* results, dvo_b200_iteration_stats* iteration_stats,
                              int32_t max_iteration_stats, const dvo_b200_weight_maps* maps);

/* ---- multi-hypothesis alignment: screen several initial poses per pair on the coarse levels, continue the best one -------
 * Dense Gauss-Newton has a small basin of convergence: after a fast rotation, a dropped frame or a loop-closure candidate
 * whose relative pose comes from a drifted graph, one initial estimate can end in a confident, wrong pose.  This call
 * starts pair p from k hypotheses H[p][0..k-1] (row-major 4 x 4, read as T_init), runs each of them on the coarse levels
 * first_level .. s only (s = screen_level), keeps one, and continues that one, from where its screening run ended, through
 * levels s-1 .. last_level.  With cfg->first_level = s the screening is dvo_slam's proposal validation on one level
 * (ConstraintProposalValidator with FirstLevel = LastLevel = 3), and the continuation its second stage.
 *   screening  hypothesis j runs levels first_level .. s exactly as dvo_b200_match_batch does with T_init = H[p][j], the
 *              same cfg except last_level = s.  Let L be that run's dvo_b200_level_stats of level s.
 *   score      j is eligible iff L.has_iteration_with_increment, ratio = L.last_increment_valid_constraints / L.valid_pixels
 *              >= min_constraint_ratio (fp64, as dvo_slam's ConstraintRatioVoter), and score =
 *              L.last_increment_log_likelihood / L.last_increment_valid_constraints, the per-constraint negative
 *              log-likelihood, is finite.  Lower is better.
 *   choice     best[p] is the eligible j with the smallest score, the lowest j on a tie; 0 if none is eligible (then every
 *              score of the pair is NaN).
 * Results, bit for bit, for every estimator, mask, batch size and launch plan:
 *   results[p] and pair p's iteration log are those of dvo_b200_match_batch of that pair alone with T_init = H[p][best[p]]
 *              (every field, the statistics of the screening levels included);
 *   screen_results[p * k + j] (optional) are those of dvo_b200_match_batch with last_level = s and T_init = H[p][j];
 *   scores[p * k + j] (optional) are the scores above, NaN where j is not eligible.
 * Cost: the screening aligns n * k pairs on the coarse levels, the continuation n pairs on the fine ones; a coarse level has a
 * quarter of the pixels of the next finer one.  Reference-role and both-role masks, cfg->mu and mixed intrinsics are
 * supported as by dvo_b200_match_batch; the photometric mode, motion priors and weight maps through
 * dvo_b200_match_batch_hypotheses_modes below.
 * Outputs in device memory and several GPUs: dvo_b200_match_batch_modes_device and _modes_sharded below. */
#define DVO_B200_MAX_HYPOTHESES 64

/* hypotheses: n * k * 16 doubles, H[p][j] at (p * k + j) * 16.  results, best: n each.  scores: n * k or NULL.
 * screen_results: n * k or NULL.  iteration_stats / max_iteration_stats as in dvo_b200_match_batch (the continued alignment's
 * log).  Refused with DVO_B200_ERR_INVALID_ARGUMENT, and dvo_b200_last_error set, before anything is staged, uploaded or
 * launched: a NULL hypotheses, results or best; k outside [1, DVO_B200_MAX_HYPOTHESES]; cfg->use_initial_estimate == 0 (the
 * hypotheses are the initial estimates); screen_level outside [cfg->last_level, cfg->first_level]; a min_constraint_ratio
 * that is not finite or lies outside [0, 1]; a hypothesis with a non-finite entry or a bottom row other than (0, 0, 0, 1);
 * and everything dvo_b200_match_batch refuses for the same n pairs.  Synchronises as dvo_b200_match_batch does. */
int dvo_b200_match_batch_hypotheses(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                                    dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents, int32_t k,
                                    const double* hypotheses, int32_t screen_level, double min_constraint_ratio,
                                    dvo_b200_result* results, int32_t* best, double* scores, dvo_b200_result* screen_results,
                                    dvo_b200_iteration_stats* iteration_stats, int32_t max_iteration_stats);

/* Multi-hypothesis alignment in the photometric mode, with motion priors and with weight maps.  The arguments of
 * dvo_b200_match_batch_hypotheses, plus, each optional:
 *   prior_information   n * k * 36 doubles or NULL: Lambda[p][j], the prior information of hypothesis j of pair p, at
 *                       (p * k + j) * 36.  Requires cfg->mu == 0.
 *   photometric_init    n * k * 2 doubles or NULL (= (1, 0) each): (alpha, beta)_0[p][j].  Only with photometric.
 *   photometric         n * 2 doubles out, or NULL: non-NULL selects the photometric mode; the final (alpha, beta) of pair p.
 *   screen_photometric  n * k * 2 doubles out, or NULL: (alpha, beta) where screening run (p, j) ended.  Only with photometric.
 *   maps                NULL (no maps) or the weight maps of the continued alignments, as dvo_b200_match_batch_maps writes them.
 * Let E be the single-pair entry point of the mode: dvo_b200_match_batch_prior with a prior (photometric as given),
 * otherwise dvo_b200_match_batch_photometric or dvo_b200_match_batch.  Bit for bit, for both estimators, every mask role
 * set, mixed intrinsics, every batch size and position and every launch plan:
 *   screening     run (p, j) is E of that pair with last_level = s from T_init = H[p][j], Lambda[p][j] and
 *                 (alpha, beta)_0[p][j]; screen_results[p * k + j] and screen_photometric[p * k + j] are what that call returns.
 *   score, choice exactly as above: the per-constraint negative log-likelihood of the data term alone.  The prior term is
 *                 not part of the score, so a hypothesis cannot win by its own prior: a tight Lambda about a wrong start
 *                 does not make that start look better.
 *   continuation  results[p], photometric[p] and pair p's iteration log are what E returns for pair p alone from the chosen
 *                 triple (H, Lambda, (alpha, beta)_0)[p][best[p]] with the call's last_level.
 *   maps          the maps, estimate and precision are what dvo_b200_match_batch_maps returns for that same single call, also
 *                 when s = last_level.
 * The prior of run (p, j) is anchored where dvo_b200_match_batch_prior anchors it, at the run's own initial estimate
 * T0 = H[p][j]; that is why Lambda is given per hypothesis.  An IMU prediction carries its Sigma^-1, a constant-velocity
 * prediction the information of the alignment it extrapolates, a zero-motion or relocalisation start 0.
 * Refused with DVO_B200_ERR_INVALID_ARGUMENT, and dvo_b200_last_error set, before anything is staged, uploaded or launched:
 * everything dvo_b200_match_batch_hypotheses refuses (checked first); photometric_init or screen_photometric without
 * photometric; with a prior, cfg->mu != 0 and a Lambda[p][j] that dvo_b200_match_batch_prior would refuse; a non-finite
 * photometric_init; with maps, everything dvo_b200_match_batch_maps refuses of its maps.  The messages name the hypothesis
 * ("hypothesis j of pair p").  dvo_b200_match_batch_hypotheses is this call with every new argument NULL.  One kernel
 * launch more with maps (k_weight_maps); synchronises once, as dvo_b200_match_batch does. */
int dvo_b200_match_batch_hypotheses_modes(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                                          dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents, int32_t k,
                                          const double* hypotheses, int32_t screen_level, double min_constraint_ratio,
                                          const double* prior_information, const double* photometric_init, double* photometric,
                                          double* screen_photometric, dvo_b200_result* results, int32_t* best, double* scores,
                                          dvo_b200_result* screen_results, dvo_b200_iteration_stats* iteration_stats,
                                          int32_t max_iteration_stats, const dvo_b200_weight_maps* maps);

/* ---- every mode with its outputs in device memory, and over several GPUs --------------------------------------------------
 * The arguments of dvo_b200_match_batch_hypotheses_modes, with k = 0 allowed.  k = 0: one plain alignment per pair;
 * hypotheses is then T_init (n * 16 doubles or NULL), prior_information n * 36 doubles and photometric_init 2n; screen_level
 * and min_constraint_ratio are ignored; best, scores, screen_results and screen_photometric must be NULL.  Let E be the
 * call the arguments stand for: for k >= 1 dvo_b200_match_batch_hypotheses_modes; for k = 0 by what is non-NULL, maps ->
 * dvo_b200_match_batch_maps, else prior_information -> _prior, else photometric -> _photometric, else dvo_b200_match_batch.
 * Every output is, byte for byte, what E returns on one context with the same arguments, for both estimators, every mask
 * role set, mixed intrinsics, every batch size and every launch plan.
 * Refused with DVO_B200_ERR_INVALID_ARGUMENT (DVO_B200_ERR_SHAPE_MISMATCH where E returns it), the last error set, before
 * anything is staged or launched: everything E refuses, first and in E's order (E's batch checks over the whole batch
 * included); for k = 0 an output only k >= 1 writes, and photometric_init without photometric; then the form's own
 * checks below.  The messages name the pair, and the hypothesis when there is one. */

/* The outputs in device memory: every output pointer is device or managed memory of the context's device, maps included,
 * which must be DVO_B200_MAPS_DEVICE.  The inputs (hypotheses / T_init, priors, photometric_init) are host memory and
 * staged as by E; the caller may free them when the call returns.  The call may wait for the context's earlier work before
 * staging; it enqueues its own work and returns without waiting for it, and copies nothing to the host
 * (dvo_b200_d2h_bytes does not move; dvo_b200_h2d_bytes and dvo_b200_kernel_launches move as for E).  A level-kernel
 * timeout surfaces at dvo_b200_synchronize.  Its own refusals, after E's: maps in DVO_B200_MAPS_HOST; then, per output in
 * argument order, a pointer not aligned to its element, and a first or last byte that cudaPointerGetAttributes does not
 * report as device or managed memory of the context's device.  dvo_b200_match_batch_device is this call with k = 0, every
 * mode argument NULL and only results. */
int dvo_b200_match_batch_modes_device(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                                      dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents, int32_t k,
                                      const double* hypotheses, int32_t screen_level, double min_constraint_ratio,
                                      const double* prior_information, const double* photometric_init, double* photometric,
                                      double* screen_photometric, dvo_b200_result* results, int32_t* best, double* scores,
                                      dvo_b200_result* screen_results, dvo_b200_iteration_stats* iteration_stats,
                                      int32_t max_iteration_stats, const dvo_b200_weight_maps* maps);
/* Over the shards of s (one context and host thread per device), outputs in host memory; maps, if given, must be
 * DVO_B200_MAPS_HOST.  Pairs are split by dvo_b200_shard_range, and pair p takes onto its shard its k hypotheses, priors
 * and photometric_init rows, its slice of every output (results, best, scores, screen_results, photometric,
 * screen_photometric, iteration_stats at p * max_iteration_stats) and its maps (planes at data + p * image_bytes, estimate,
 * precision).  Each shard runs E on its own context, with that context's estimator; a pair's bits do not depend on its
 * batch, so with the same estimator everywhere the outputs are E's on one context.  The whole batch is checked before any
 * shard starts, so a refusal leaves every shard's context untouched: after E's checks, a pair whose pyramids do not live on
 * the device of the shard that owns it, then maps in DVO_B200_MAPS_DEVICE.  Returns once every shard is done. */
int dvo_b200_match_batch_modes_sharded(dvo_b200_sharded* s, const dvo_b200_config* cfg, int32_t n,
                                       dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents, int32_t k,
                                       const double* hypotheses, int32_t screen_level, double min_constraint_ratio,
                                       const double* prior_information, const double* photometric_init, double* photometric,
                                       double* screen_photometric, dvo_b200_result* results, int32_t* best, double* scores,
                                       dvo_b200_result* screen_results, dvo_b200_iteration_stats* iteration_stats,
                                       int32_t max_iteration_stats, const dvo_b200_weight_maps* maps);

/* ---- profiling hooks (bench.py roofline): per-kernel-class accumulated device time measured with
 *      CUDA events on the ctx stream.  classes: 0 residual/scale stage, 1 normal-equation stage,
 *      2 per-pair step kernels, 3 pyramid build, 4 selection. -------------------------------- */
int dvo_b200_profile_enable(dvo_b200_ctx* ctx, int32_t enable);
int dvo_b200_profile_read(dvo_b200_ctx* ctx, double ms_out[8], int64_t launches_out[8], int32_t reset);

#ifdef __cplusplus
}
#endif
#endif /* DVO_B200_H_ */
