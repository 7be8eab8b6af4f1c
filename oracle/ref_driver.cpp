// ref_driver.cpp -- TEST INFRASTRUCTURE.  Drives the REFERENCE'S OWN compiled functions (oracle/_ref/, built by
// `make -C oracle ref REF=<dvo_slam checkout>/dvo_core` from src/{dense_tracking_impl,core/math_sse,core/intrinsic_matrix}.cpp,
// unmodified, against the header-only shims in oracle/ref_shim/) through one Gauss-Newton linearisation exactly as
// DenseTracker::match() strings them together (dense_tracking.cpp:212-220, 271-343), so that the oracle's FAITHFUL
// mode can be checked bit for bit against reference-produced numbers (tests/test_reference_pin.py).
//
// What comes from the reference's object code: computeResidualsSse, computeWeightsSse, computeScaleSse,
// computeCompleteDataLogLikelihood (dense_tracking_impl.cpp), OptimizedSelfAdjointMatrix6x6f::rankUpdate / toEigen
// (math_sse.cpp), IntrinsicMatrix (intrinsic_matrix.cpp), ValidPointAndGradientThresholdPredicate::isPointOk
// (point_selection.h, inline).  What this file restates because its translation unit needs OpenCV / Sophus proper
// (each block cites its lines): the acceleration image (rgbd_image.cpp:534-543), the point cloud
// (rgbd_image.cpp:186-204, 245-262), the point list (point_selection.cpp:119-152), the residual weight vectors
// (dense_tracking.cpp:215-220), the Jacobians (dense_tracking.cpp:448-476) and the three lines of
// NormalEquationsLeastSquares::update/finish (least_squares.cpp:58-64, 74-80).
#include <dvo/dense_tracking_impl.h>

#include <cstdint>
#include <cstring>
#include <vector>

namespace dvo {
namespace core {
// link stubs for the two constructors the driver needs (rgbd_image.cpp:186-204, 320-332; the template cloud is built below)
RgbdCamera::RgbdCamera(size_t width, size_t height, const IntrinsicMatrix& intrinsics) : width_(width), height_(height), intrinsics_(intrinsics) {}
RgbdCamera::~RgbdCamera() {}
RgbdImage::RgbdImage(const RgbdCamera& camera)
    : width(0), height(0), intensity_requires_calculation_(true), depth_requires_calculation_(true), pointcloud_requires_build_(true), camera_(camera) {}
RgbdImage::~RgbdImage() {}
bool RgbdImage::inImage(const float& x, const float& y) const { return x >= 0 && x < width && y >= 0 && y < height; }   // rgbd_image.cpp (only the scalar twin calls it)
}  // namespace core
}  // namespace dvo

using namespace dvo::core;

extern "C" {

// planes6: I, Z, Ix, Iy, Zx, Zy (h*w floats each).  ti / td: DenseTracker::Config::Intensity/DepthDerivativeThreshold.
// Outputs: n_selected, n (valid constraints), residuals (2 floats per valid point, list order), point index (linear
// pixel index of every valid point), weights, P (row-major 2x2), ll, A (row-major 6x6 float), b (6 floats).
int64_t ref_linearize(const float* ref_planes6, const float* cur_planes6, int w, int h, const float K4[4], const double T[16], float ti,
                      float td, int use_weights, const float prev_precision[4], int64_t* n_selected, float* residuals_out,
                      int32_t* index_out, float* records_out, float* weights_out, float P_out[4], float* ll_out, float A_out[36],
                      float b_out[6]) {
  const size_t N = (size_t)w * h;
  IntrinsicMatrix K = IntrinsicMatrix::create(K4[0], K4[1], K4[2], K4[3]);
  RgbdCamera camera(w, h, K);
  RgbdImage current(camera);
  current.width = w; current.height = h;
  // buildAccelerationStructure (rgbd_image.cpp:534-543): cv::merge of {intensity, depth, idx, idy, zdx, zdy, 0, 0}
  current.acceleration = cv::Mat_<RgbdImage::Vec8f>(h, w);
  for (size_t i = 0; i < N; ++i) {
    float* a = current.acceleration.ptr<float>(0) + 8 * i;
    for (int c = 0; c < 6; ++c) a[c] = cur_planes6[c * N + i];
    a[6] = 0.f; a[7] = 0.f;
  }
  // reference point list: point cloud (rgbd_image.cpp:186-204, 245-262) + selectPointsFromImage (point_selection.cpp:119-152)
  ValidPointAndGradientThresholdPredicate predicate;
  predicate.intensity_threshold = ti; predicate.depth_threshold = td;
  PointWithIntensityAndDepth::VectorType points;
  std::vector<int32_t> point_index;
  {
    size_t idx = 0;
    for (size_t y = 0; y < (size_t)h; ++y)
      for (size_t x = 0; x < (size_t)w; ++x, ++idx) {
        const float tx = (x - K.ox()) / K.fx(), ty = (y - K.oy()) / K.fy();
        const float depth = ref_planes6[1 * N + idx];
        PointWithIntensityAndDepth p;
        p.point.data[0] = tx * depth; p.point.data[1] = ty * depth; p.point.data[2] = 1.0f * depth; p.point.data[3] = 1.0f;
        for (int c = 0; c < 6; ++c) p.intensity_and_depth.data[c] = ref_planes6[c * N + idx];
        p.intensity_and_depth.data[6] = 0.f; p.intensity_and_depth.data[7] = 0.f;
        if (predicate.isPointOk(x, y, p.point.z, p.intensity_and_depth.idx, p.intensity_and_depth.idy, p.intensity_and_depth.zdx, p.intensity_and_depth.zdy)) {
          points.push_back(p);
          point_index.push_back((int32_t)idx);
        }
      }
  }
  *n_selected = (int64_t)points.size();
  // dense_tracking.cpp:215-220
  Vector8f wcur, wref;
  float wcur_id = 0.5f, wref_id = 0.5f, wcur_zd = 1.0f, wref_zd = 0.0f;
  wcur <<  1.0f / 255.0f,  1.0f, wcur_id * K.fx() / 255.0f, wcur_id * K.fy() / 255.0f, wcur_zd * K.fx(), wcur_zd * K.fy(), 0.0f, 0.0f;
  wref << -1.0f / 255.0f, -1.0f, wref_id * K.fx() / 255.0f, wref_id * K.fy() / 255.0f, wref_zd * K.fx(), wref_zd * K.fy(), 0.0f, 0.0f;
  // dense_tracking.cpp:263: transformf = estimate.cast<float>()
  Eigen::Affine3f transformf;
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) transformf(i, j) = (float)T[i * 4 + j];

  PointWithIntensityAndDepth::VectorType points_error(points.size() + 2);
  dvo::DenseTracker::ResidualVectorType residuals(points.size() + 2);
  dvo::DenseTracker::WeightVectorType weights(points.size() + 2);
  ComputeResidualsResult rr;
  rr.first_point_error = points_error.begin();
  rr.first_residual = residuals.begin();
  computeResidualsSse(points.begin(), points.end(), current, K, transformf, wref, wcur, rr);      // dense_tracking.cpp:271
  const size_t n = rr.last_residual - rr.first_residual;
  Eigen::Vector2f mean; mean.setZero();
  Eigen::Matrix2f precision;
  for (int i = 0; i < 2; ++i) for (int j = 0; j < 2; ++j) precision(i, j) = prev_precision ? prev_precision[i * 2 + j] : 0.f;
  if (!use_weights) std::fill(weights.begin(), weights.begin() + n, 1.0f);                         // dense_tracking.cpp:286-293
  else computeWeightsSse(rr.first_residual, rr.last_residual, weights.begin(), mean, precision);
  precision = computeScaleSse(rr.first_residual, rr.last_residual, weights.begin(), mean).inverse();   // :295
  const float ll = computeCompleteDataLogLikelihood(rr.first_residual, rr.last_residual, weights.begin(), mean, precision);   // :297

  // dense_tracking.cpp:327-343 with NormalEquationsLeastSquares::update / finish (least_squares.cpp:58-64, 74-80)
  OptimizedSelfAdjointMatrix6x6f A_opt;
  A_opt.setZero();
  Vector6 b; b.setZero();
  {
    dvo::DenseTracker::WeightVectorType::iterator w_it = weights.begin();
    for (PointIterator e_it = rr.first_point_error; e_it != rr.last_point_error; ++e_it, ++w_it) {
      const float* p = e_it->point.data;
      Matrix2x6 Jw, J;
      Vector6 Jz;
      // computeJacobianOfProjectionAndTransformation (dense_tracking.cpp:448-466)
      NumType z = 1.0f / p[2];
      NumType z_sqr = 1.0f / (p[2] * p[2]);
      Jw(0, 0) = z; Jw(0, 1) = 0.0f; Jw(0, 2) = -p[0] * z_sqr; Jw(0, 3) = Jw(0, 2) * p[1]; Jw(0, 4) = 1.0f - Jw(0, 2) * p[0]; Jw(0, 5) = -p[1] * z;
      Jw(1, 0) = 0.0f; Jw(1, 1) = z; Jw(1, 2) = -p[1] * z_sqr; Jw(1, 3) = -1.0f + Jw(1, 2) * p[1]; Jw(1, 4) = -Jw(0, 3); Jw(1, 5) = p[0] * z;
      // compute3rdRowOfJacobianOfTransformation (dense_tracking.cpp:468-476)
      Jz(0) = 0.0; Jz(1) = 0.0; Jz(2) = 1.0; Jz(3) = p[1]; Jz(4) = -p[0]; Jz(5) = 0.0;
      // J.row(0) = intensity derivative^T * Jw;  J.row(1) = depth derivative^T * Jw - Jz^T   (dense_tracking.cpp:338-339)
      const float* e = e_it->intensity_and_depth.data;
      for (int c = 0; c < 6; ++c) {
        J(0, c) = e[2] * Jw(0, c) + e[3] * Jw(1, c);
        J(1, c) = (e[4] * Jw(0, c) + e[5] * Jw(1, c)) - Jz(c);
      }
      Eigen::Vector2f r(e[0], e[1]);
      Eigen::Matrix2f W = (*w_it) * precision;
      A_opt.rankUpdate(J, W);                        // least_squares.cpp:60 -> math_sse.cpp:82-178
      b -= J.transpose() * W * r;                    // least_squares.cpp:61
    }
  }
  Matrix6x6 A;
  A_opt.toEigen(A);                                  // least_squares.cpp:76

  for (size_t i = 0; i < n; ++i) {
    if (residuals_out) { residuals_out[2 * i] = residuals[i](0); residuals_out[2 * i + 1] = residuals[i](1); }
    if (weights_out) weights_out[i] = weights[i];
    if (records_out) std::memcpy(records_out + 12 * i, &points_error[i], sizeof(float) * 12);
  }
  if (index_out) {
    // computeResidualsSse copies the reference point (x, y, z, 1) into every valid record: recover its pixel by walking
    // the selected list in order (records keep the list order)
    size_t k = 0;
    for (size_t i = 0; i < n; ++i) {
      while (k < points.size() && std::memcmp(points[k].point.data, points_error[i].point.data, sizeof(float) * 4) != 0) ++k;
      index_out[i] = k < points.size() ? point_index[k] : -1;
      ++k;
    }
  }
  if (P_out) for (int i = 0; i < 2; ++i) for (int j = 0; j < 2; ++j) P_out[i * 2 + j] = precision(i, j);
  if (ll_out) *ll_out = ll;
  if (A_out) for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) A_out[i * 6 + j] = A(i, j);
  if (b_out) for (int i = 0; i < 6; ++i) b_out[i] = b(i);
  return (int64_t)n;
}


// ---- whole alignments through the reference's object code ----------------------------------------------------------------
// ref_match() is DenseTracker::match() (dense_tracking.cpp:131-376) with every per-point pass executed by the reference's
// own compiled functions and data structures (no conversions inside the loop): the control flow, the Revertable poses and the
// statistics are restated here (dense_tracking.cpp itself needs Sophus); SE(3) exp/log and the 6x6 LDL^T come from the
// oracle (orc_se3_exp / orc_se3_log / orc_ldlt_solve6, which restate Sophus / Eigen).  Used as the CPU baseline of bench.py
// (kind "reference") and by tests/test_reference_pin.py (control flow and pose equal to the oracle's FAITHFUL mode).
void orc_se3_exp(const double xi[6], double T[16]);
void orc_se3_log(const double T[16], double xi[6]);
void orc_ldlt_solve6(const double A[36], const double b[6], double x[6]);

}  // extern "C"

namespace {

struct RefLevel {
  int w = 0, h = 0;
  IntrinsicMatrix K;
  RgbdCamera* camera = nullptr;
  RgbdImage* image = nullptr;                         // carries the acceleration image (rgbd_image.cpp:534-543)
  std::vector<float> depth;                           // for the point cloud of the reference role
  PointWithIntensityAndDepth::VectorType points;      // PointSelection's cached list (point_selection.cpp:100-113)
  float ti = -1.f, td = -1.f;
  bool have_points = false;
};
struct RefPyramid {
  std::vector<RefLevel> levels;
  ~RefPyramid() { for (RefLevel& l : levels) { delete l.image; delete l.camera; } }
};

void select_points(RefLevel& L, float ti, float td) {
  if (L.have_points && L.ti == ti && L.td == td) return;
  ValidPointAndGradientThresholdPredicate predicate;
  predicate.intensity_threshold = ti; predicate.depth_threshold = td;
  L.points.clear();
  const float* accel = L.image->acceleration.ptr<float>(0);
  size_t idx = 0;
  for (size_t y = 0; y < (size_t)L.h; ++y)
    for (size_t x = 0; x < (size_t)L.w; ++x, ++idx) {
      const float tx = (x - L.K.ox()) / L.K.fx(), ty = (y - L.K.oy()) / L.K.fy();   // rgbd_image.cpp:197-198
      const float depth = L.depth[idx];
      PointWithIntensityAndDepth p;
      p.point.data[0] = tx * depth; p.point.data[1] = ty * depth; p.point.data[2] = 1.0f * depth; p.point.data[3] = 1.0f;   // :258-259
      std::memcpy(p.intensity_and_depth.data, accel + 8 * idx, sizeof(float) * 8);
      if (predicate.isPointOk(x, y, p.point.z, p.intensity_and_depth.idx, p.intensity_and_depth.idy, p.intensity_and_depth.zdx, p.intensity_and_depth.zdy))
        L.points.push_back(p);
    }
  L.ti = ti; L.td = td; L.have_points = true;
}

// rigid 4x4 (row-major double) helpers
void mat_mul(const double A[16], const double B[16], double C[16]) {
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += A[i * 4 + k] * B[k * 4 + j]; C[i * 4 + j] = s; }
}
void mat_inv(const double A[16], double B[16]) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) B[i * 4 + j] = A[j * 4 + i];
  for (int i = 0; i < 3; ++i) { double s = 0; for (int k = 0; k < 3; ++k) s += A[k * 4 + i] * A[k * 4 + 3]; B[i * 4 + 3] = -s; }
  B[12] = B[13] = B[14] = 0; B[15] = 1;
}
void mat_identity(double A[16]) { for (int i = 0; i < 16; ++i) A[i] = (i % 5 == 0) ? 1.0 : 0.0; }

}  // namespace

extern "C" {

void* ref_pyramid_create(int nlevels, const float* const* planes6, const int* w, const int* h, const float* K4) {
  RefPyramid* P = new RefPyramid;
  P->levels.resize(nlevels);
  for (int l = 0; l < nlevels; ++l) {
    RefLevel& L = P->levels[l];
    L.w = w[l]; L.h = h[l];
    L.K = IntrinsicMatrix::create(K4[4 * l], K4[4 * l + 1], K4[4 * l + 2], K4[4 * l + 3]);
    L.camera = new RgbdCamera(L.w, L.h, L.K);
    L.image = new RgbdImage(*L.camera);
    L.image->width = L.w; L.image->height = L.h;
    const size_t N = (size_t)L.w * L.h;
    L.image->acceleration = cv::Mat_<RgbdImage::Vec8f>(L.h, L.w);
    float* a = L.image->acceleration.ptr<float>(0);
    for (size_t i = 0; i < N; ++i) {
      for (int c = 0; c < 6; ++c) a[8 * i + c] = planes6[l][c * N + i];
      a[8 * i + 6] = 0.f; a[8 * i + 7] = 0.f;
    }
    L.depth.assign(planes6[l] + N, planes6[l] + 2 * N);
  }
  return P;
}
void ref_pyramid_destroy(void* p) { delete static_cast<RefPyramid*>(p); }

// DenseTracker::computeIntensityErrorImage (dense_tracking.cpp:378-444) with the residuals AND the valid flags produced by
// the reference's own computeResidualsAndValidFlagsSse (the Debug instantiation of the SSE loop); the raster walk over the
// selection's debug index is restated from lines 415-439.  image: h*w floats.  Returns the residuals consumed.
int64_t ref_intensity_error_image(void* ref_p, void* cur_p, int level, const double* T, float ti, float td, float* image) {
  RefPyramid& ref = *static_cast<RefPyramid*>(ref_p);
  RefPyramid& cur = *static_cast<RefPyramid*>(cur_p);
  RefLevel& R = ref.levels[level];
  RefLevel& C = cur.levels[level];
  select_points(R, ti, td);
  const size_t N = (size_t)R.w * R.h;
  // debug index: 1 at every selected pixel (point_selection.cpp:139-140); same predicate walk as select_points()
  std::vector<uint8_t> debug_idx(N, 0);
  {
    ValidPointAndGradientThresholdPredicate predicate;
    predicate.intensity_threshold = ti; predicate.depth_threshold = td;
    const float* accel = R.image->acceleration.ptr<float>(0);
    size_t idx = 0;
    for (size_t y = 0; y < (size_t)R.h; ++y)
      for (size_t x = 0; x < (size_t)R.w; ++x, ++idx) {
        const float* a = accel + 8 * idx;
        if (predicate.isPointOk(x, y, R.depth[idx], a[2], a[3], a[4], a[5])) debug_idx[idx] = 1;
      }
  }
  const IntrinsicMatrix& K = C.K;
  Vector8f wcur, wref;                                 // dense_tracking.cpp:401-406
  float wcur_id = 0.5f, wref_id = 0.5f, wcur_zd = 1.0f, wref_zd = 0.0f;
  wcur <<  1.0f / 255.0f,  1.0f, wcur_id * K.fx() / 255.0f, wcur_id * K.fy() / 255.0f, wcur_zd * K.fx(), wcur_zd * K.fy(), 0.0f, 0.0f;
  wref << -1.0f / 255.0f, -1.0f, wref_id * K.fx() / 255.0f, wref_id * K.fy() / 255.0f, wref_zd * K.fx(), wref_zd * K.fy(), 0.0f, 0.0f;
  Eigen::Affine3f transformf;
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) transformf(i, j) = (float)T[i * 4 + j];   // transformation.cast<float>() (:413)
  PointWithIntensityAndDepth::VectorType points_error(R.points.size() + 2);
  dvo::DenseTracker::ResidualVectorType residuals(R.points.size() + 2);
  std::vector<uint8_t> valid_residuals;
  valid_residuals.resize(R.points.size() + 2);          // zero-initialised, as line 391
  ComputeResidualsResult rr;
  rr.first_point_error = points_error.begin();
  rr.first_residual = residuals.begin();
  rr.first_valid_flag = valid_residuals.begin();
  computeResidualsAndValidFlagsSse(R.points.begin(), R.points.end(), *C.image, K, transformf, wref, wcur, rr);
  for (size_t i = 0; i < N; ++i) image[i] = 0.0f;
  const uint8_t* valid_pixel_it = debug_idx.data();
  ValidFlagIterator valid_residual_it = rr.first_valid_flag;
  ResidualIterator residual_it = rr.first_residual;
  for (size_t i = 0; i < N; ++i, ++valid_pixel_it) {   // lines 426-439
    if (*valid_pixel_it == 1) {
      if (*valid_residual_it == 1) {
        image[i] = std::abs(residual_it->coeff(0));
        ++residual_it;
      }
      ++valid_residual_it;
    }
  }
  return (int64_t)(residual_it - rr.first_residual);
}

// termination codes as dvo::DenseTracker::TerminationCriteria (dense_tracking.h:71-81):
// 0 IterationsExceeded, 1 IncrementTooSmall, 2 LogLikelihoodDecreased, 3 TooFewConstraints
int ref_match(void* ref_p, void* cur_p, int first_level, int last_level, int max_iterations, double precision_cfg, double mu,
              int use_initial_estimate, const double* T_init, float ti, float td, double T_out[16], double info_out[36],
              double* ll_out, int32_t* termination, int32_t* num_iterations, int64_t* valid_pixels) {
  RefPyramid& ref = *static_cast<RefPyramid*>(ref_p);
  RefPyramid& cur = *static_cast<RefPyramid*>(cur_p);
  // DenseTracker members (dense_tracking.cpp:160-165)
  static thread_local PointWithIntensityAndDepth::VectorType points_error;
  static thread_local dvo::DenseTracker::ResidualVectorType residuals;
  static thread_local dvo::DenseTracker::WeightVectorType weights;

  double inc[16], initial[16], initial_old[16], estimate[16], estimate_old[16];
  if (use_initial_estimate && T_init) std::memcpy(inc, T_init, sizeof(inc)); else mat_identity(inc);       // :137-147
  std::memcpy(initial, inc, sizeof(inc)); std::memcpy(initial_old, inc, sizeof(inc));
  mat_identity(estimate); mat_identity(estimate_old);
  bool accept = true;
  const double kNaN = std::numeric_limits<double>::quiet_NaN();
  double A_last[36], A_prev[36], nll_last = kNaN, nll_prev = kNaN, prior_last = 0, prior_prev = 0;
  int have = 0;       // completed iterations recorded on the last level (0, 1, 2+)
  int li = 0, last_termination = -1, last_level_iterations = 0;
  for (int level = first_level; level >= last_level; --level, ++li) {
    RefLevel& R = ref.levels[level];
    RefLevel& C = cur.levels[level];
    Eigen::Vector2f mean; mean.setZero();
    Eigen::Matrix2f precision; precision.setZero();                                  // :205-206
    int iteration = 0;
    double error = std::numeric_limits<double>::max(), last_error = error;
    select_points(R, ti, td);                                                        // :225
    valid_pixels[li] = (int64_t)R.points.size();
    if (points_error.size() < R.points.size() + 2) { points_error.resize(R.points.size() + 2); residuals.resize(R.points.size() + 2); weights.resize(R.points.size() + 2); }
    Vector8f wcur, wref;                                                             // :215-220
    float wcur_id = 0.5f, wref_id = 0.5f, wcur_zd = 1.0f, wref_zd = 0.0f;
    const IntrinsicMatrix& K = C.K;
    wcur <<  1.0f / 255.0f,  1.0f, wcur_id * K.fx() / 255.0f, wcur_id * K.fy() / 255.0f, wcur_zd * K.fx(), wcur_zd * K.fy(), 0.0f, 0.0f;
    wref << -1.0f / 255.0f, -1.0f, wref_id * K.fx() / 255.0f, wref_id * K.fy() / 255.0f, wref_zd * K.fx(), wref_zd * K.fy(), 0.0f, 0.0f;
    double x[6];
    orc_se3_log(inc, x);                                                             // :238
    int term = -1, recorded = 0;
    have = 0;
    do {
      orc_se3_exp(x, inc);                                                           // :259
      double inv[16], tmp[16];
      mat_inv(inc, inv);
      std::memcpy(initial_old, initial, sizeof(initial)); mat_mul(inv, initial, tmp); std::memcpy(initial, tmp, sizeof(tmp));      // :260
      std::memcpy(estimate_old, estimate, sizeof(estimate)); mat_mul(inc, estimate, tmp); std::memcpy(estimate, tmp, sizeof(tmp));   // :261
      Eigen::Affine3f transformf;
      for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) transformf(i, j) = (float)estimate[i * 4 + j];                        // :263
      ComputeResidualsResult rr;
      rr.first_point_error = points_error.begin();
      rr.first_residual = residuals.begin();
      computeResidualsSse(R.points.begin(), R.points.end(), *C.image, K, transformf, wref, wcur, rr);                               // :271
      const size_t n = rr.last_residual - rr.first_residual;
      ++recorded;
      if (n < 6) {                                                                   // :276-284
        std::memcpy(initial, initial_old, sizeof(initial)); std::memcpy(estimate, estimate_old, sizeof(estimate));
        term = 3;
        break;
      }
      if (iteration == 0) std::fill(weights.begin(), weights.begin() + n, 1.0f);    // :286-293
      else computeWeightsSse(rr.first_residual, rr.last_residual, weights.begin(), mean, precision);
      precision = computeScaleSse(rr.first_residual, rr.last_residual, weights.begin(), mean).inverse();                           // :295
      const float ll = computeCompleteDataLogLikelihood(rr.first_residual, rr.last_residual, weights.begin(), mean, precision);     // :297
      double li6[6];
      orc_se3_log(initial, li6);
      double sq = 0;
      for (int i = 0; i < 6; ++i) sq += li6[i] * li6[i];
      const double prior = mu * sq;                                                  // :302
      last_error = error;                                                            // :306-307
      error = -(double)ll;
      accept = error < last_error;                                                   // :312
      if (!accept) {
        std::memcpy(initial, initial_old, sizeof(initial)); std::memcpy(estimate, estimate_old, sizeof(estimate));
        term = 2;
        break;
      }
      // :327-343
      OptimizedSelfAdjointMatrix6x6f A_opt;
      A_opt.setZero();
      Vector6 b; b.setZero();
      dvo::DenseTracker::WeightVectorType::iterator w_it = weights.begin();
      for (PointIterator e_it = rr.first_point_error; e_it != rr.last_point_error; ++e_it, ++w_it) {
        const float* p = e_it->point.data;
        Matrix2x6 Jw, J;
        NumType z = 1.0f / p[2];
        NumType z_sqr = 1.0f / (p[2] * p[2]);
        Jw(0, 0) = z; Jw(0, 1) = 0.0f; Jw(0, 2) = -p[0] * z_sqr; Jw(0, 3) = Jw(0, 2) * p[1]; Jw(0, 4) = 1.0f - Jw(0, 2) * p[0]; Jw(0, 5) = -p[1] * z;
        Jw(1, 0) = 0.0f; Jw(1, 1) = z; Jw(1, 2) = -p[1] * z_sqr; Jw(1, 3) = -1.0f + Jw(1, 2) * p[1]; Jw(1, 4) = -Jw(0, 3); Jw(1, 5) = p[0] * z;
        const float Jz[6] = {0.0f, 0.0f, 1.0f, p[1], -p[0], 0.0f};
        const float* e = e_it->intensity_and_depth.data;
        for (int c = 0; c < 6; ++c) {
          J(0, c) = e[2] * Jw(0, c) + e[3] * Jw(1, c);
          J(1, c) = (e[4] * Jw(0, c) + e[5] * Jw(1, c)) - Jz[c];
        }
        Eigen::Vector2f r(e[0], e[1]);
        Eigen::Matrix2f W = (*w_it) * precision;
        A_opt.rankUpdate(J, W);
        b -= J.transpose() * W * r;
      }
      Matrix6x6 Af;
      A_opt.toEigen(Af);
      double A[36], bd[6];
      for (int i = 0; i < 6; ++i) { for (int j = 0; j < 6; ++j) A[i * 6 + j] = (double)Af(i, j); bd[i] = (double)b(i); }
      for (int i = 0; i < 6; ++i) { A[i * 6 + i] += mu; bd[i] += mu * li6[i]; }      // :345-346
      orc_ldlt_solve6(A, bd, x);                                                     // :347
      std::memcpy(A_prev, A_last, sizeof(A_prev)); nll_prev = nll_last; prior_prev = prior_last;
      std::memcpy(A_last, A, sizeof(A_last)); nll_last = -(double)ll; prior_last = prior;
      ++have;
      iteration++;                                                                   // :353
      double m = 0;
      for (int i = 0; i < 6; ++i) m = std::fabs(x[i]) > m ? std::fabs(x[i]) : m;
      if (!(accept && m > precision_cfg && !(iteration >= max_iterations))) break;   // :357
    } while (true);
    {
      double m = 0;
      for (int i = 0; i < 6; ++i) m = std::fabs(x[i]) > m ? std::fabs(x[i]) : m;
      if (m <= precision_cfg) term = 1;                                              // :359
      if (iteration >= max_iterations) term = 0;                                     // :362
    }
    termination[li] = term;
    num_iterations[li] = recorded;
    last_termination = term; last_level_iterations = recorded;
  }
  // :368-373: last iteration of the last level, or the one before after LogLikelihoodDecreased
  (void)last_level_iterations;
  double inv[16];
  mat_inv(estimate, inv);
  std::memcpy(T_out, inv, sizeof(inv));
  const double* Apick = nullptr; double nll = kNaN, prior = 0;
  if (last_termination == 2) { if (have >= 1) { Apick = A_last; nll = nll_last; prior = prior_last; } }   // the rejected iteration recorded no system
  else if (last_termination != 3 && have >= 1) { Apick = A_last; nll = nll_last; prior = prior_last; }
  for (int i = 0; i < 36; ++i) info_out[i] = Apick ? Apick[i] * 0.008 * 0.008 : kNaN;
  *ll_out = Apick ? nll + prior : kNaN;
  (void)A_prev; (void)nll_prev; (void)prior_prev;
  return 0;
}

}  // extern "C"
