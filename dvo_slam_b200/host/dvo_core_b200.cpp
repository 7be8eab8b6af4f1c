// dvo_core_b200.cpp -- implementation of the adapter classes in include/dvo/ (the reference's
// libdvo_core.so surface for the hot path) on top of the C ABI of libdvo_b200.so.
#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <stdexcept>

#include "dvo/dense_tracking.h"
#include "../csrc/hypotheses_args.h"   // the checks of dvo_b200_match_batch_hypotheses[_modes], run here so that a refusal returns false
#include "../csrc/prior_args.h"   // the prior checks of dvo_b200_match_batch_prior, run here so that a refusal returns false

namespace dvo {
namespace core {

// ---- cameras (rgbd_image.cpp:186-296) -------------------------------------------------------------
RgbdImagePtr RgbdCamera::create(const cv::Mat& intensity, const cv::Mat& depth) const {
  RgbdImagePtr r(new RgbdImage(*this));
  r->intensity = intensity;
  r->depth = depth;
  r->initialize();
  return r;
}
RgbdImagePtr RgbdCamera::create() const { return RgbdImagePtr(new RgbdImage(*this)); }

RgbdCameraPyramid::RgbdCameraPyramid(const RgbdCamera& base) { levels_.push_back(RgbdCameraPtr(new RgbdCamera(base))); }
RgbdCameraPyramid::RgbdCameraPyramid(size_t w, size_t h, const IntrinsicMatrix& k) { levels_.push_back(RgbdCameraPtr(new RgbdCamera(w, h, k))); }
RgbdImagePyramidPtr RgbdCameraPyramid::create(const cv::Mat& base_intensity, const cv::Mat& base_depth) {
  return RgbdImagePyramidPtr(new RgbdImagePyramid(*this, base_intensity, base_depth));
}
void RgbdCameraPyramid::build(size_t levels) {   // rgbd_image.cpp:283-296: whole K times 0.5 per level
  for (size_t idx = levels_.size(); idx < levels; ++idx) {
    const RgbdCamera& prev = *levels_[idx - 1];
    IntrinsicMatrix k(prev.intrinsics());
    k.scale(0.5f);
    levels_.push_back(RgbdCameraPtr(new RgbdCamera(prev.width() / 2, prev.height() / 2, k)));
  }
}
const RgbdCamera& RgbdCameraPyramid::level(size_t level) { build(level + 1); return *levels_[level]; }
const RgbdCamera& RgbdCameraPyramid::level(size_t level) const { return *levels_[level]; }

// ---- image pyramid ----------------------------------------------------------------------------------
RgbdImagePyramid::RgbdImagePyramid(RgbdCameraPyramid& camera, const cv::Mat& intensity, const cv::Mat& depth)
    : camera_(camera), mask_current_(false), device_(0), device_ctx_(0), device_levels_(0), requested_levels_(1) {
  levels_.push_back(camera_.level(0).create(intensity, depth));
}
RgbdImagePyramid::~RgbdImagePyramid() {
  if (device_) dvo_b200_pyramid_release(device_);
}
void RgbdImagePyramid::build(const size_t num_levels) {
  // Coarser levels are produced on the device together with their derivatives (rgbd_image.cpp:156-172);
  // here only the request is recorded, host copies of a level are fetched on demand by level().
  if (num_levels > requested_levels_) requested_levels_ = num_levels;
  camera_.build(num_levels);
}
double RgbdImagePyramid::timestamp() const { return !levels_.empty() ? levels_[0]->timestamp : 0.0; }

bool RgbdImagePyramid::setReferenceMask(const cv::Mat& mask) { return setMask(mask, false); }

bool RgbdImagePyramid::setMask(const cv::Mat& mask, bool current_role_too) {
  std::lock_guard<std::mutex> lock(mutex_);
  const RgbdImage& l0 = *levels_[0];
  if (device_ || mask.type() != CV_8UC1 || mask.rows != l0.intensity.rows || mask.cols != l0.intensity.cols) return false;
  mask_ = mask.clone();
  mask_current_ = current_role_too;
  return true;
}

// the role set of a pyramid's mask (dvo_b200_pyramid_create_masked_batch_roles)
static int32_t mask_roles(bool current_role_too) {
  return current_role_too ? DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT : DVO_B200_MASK_ROLE_REFERENCE;
}

// the reference mask as n*h*w contiguous bytes (a cv::Mat need not be continuous), or empty without one
static void append_mask(const cv::Mat& mask, int w, int h, std::vector<uint8_t>& out) {
  const size_t base = out.size();
  out.resize(base + size_t(w) * h, 1);   // no mask: all usable, the same bits as an unmasked pyramid
  if (mask.empty()) return;
  for (int y = 0; y < h; ++y) std::memcpy(&out[base + size_t(y) * w], mask.ptr<uint8_t>(y), size_t(w));
}

dvo_b200_pyramid* RgbdImagePyramid::device(dvo_b200_ctx* ctx, size_t levels) {
  std::lock_guard<std::mutex> lock(mutex_);
  if (levels < requested_levels_) levels = requested_levels_;
  if (device_ && device_levels_ >= levels) return device_;
  if (device_) { dvo_b200_pyramid_release(device_); device_ = 0; }
  RgbdImage& l0 = *levels_[0];
  if (l0.intensity.type() != CV_32FC1 || l0.depth.type() != CV_32FC1)
    throw std::runtime_error("RgbdImagePyramid: intensity and depth must be CV_32FC1 (benchmark_slam.cpp:60-77)");
  const IntrinsicMatrix& k = camera_.level(0).intrinsics();
  std::vector<uint8_t> mask;
  if (!mask_.empty()) append_mask(mask_, l0.intensity.cols, l0.intensity.rows, mask);
  int rc = dvo_b200_pyramid_create_masked_batch_roles(ctx, 1, DVO_B200_INPUT_FLOAT32, l0.intensity.ptr<float>(), l0.depth.ptr<float>(),
                                                      0.f, mask.empty() ? nullptr : mask.data(), mask_roles(mask_current_),
                                                      l0.intensity.cols, l0.intensity.rows, k.fx(), k.fy(), k.ox(), k.oy(), int(levels),
                                                      &device_);
  if (rc != 0) throw std::runtime_error(std::string("dvo_b200_pyramid_create_masked_batch_roles: ") + dvo_b200_last_error(ctx));
  dvo_b200_synchronize(ctx);   // the host cv::Mat may be released by the caller
  device_ctx_ = ctx;
  device_levels_ = levels;
  return device_;
}

void RgbdImagePyramid::deviceBatch(dvo_b200_ctx* ctx, const std::vector<RgbdImagePyramid*>& pyramids, size_t levels,
                                   std::vector<dvo_b200_pyramid*>& out) {
  out.assign(pyramids.size(), static_cast<dvo_b200_pyramid*>(0));
  // distinct pyramids without a sufficient device mirror, of the geometry of the first such pyramid
  std::vector<RgbdImagePyramid*> todo;
  int w = 0, h = 0;
  for (size_t i = 0; i < pyramids.size(); ++i) {
    RgbdImagePyramid* p = pyramids[i];
    std::lock_guard<std::mutex> lock(p->mutex_);
    if (p->device_ && p->device_levels_ >= std::max(levels, p->requested_levels_)) continue;
    if (std::find(todo.begin(), todo.end(), p) != todo.end()) continue;
    const RgbdImage& l0 = *p->levels_[0];
    if (l0.intensity.type() != CV_32FC1 || l0.depth.type() != CV_32FC1) continue;
    if (todo.empty()) { w = l0.intensity.cols; h = l0.intensity.rows; }
    else if (l0.intensity.cols != w || l0.intensity.rows != h || &p->camera_ != &todo[0]->camera_) continue;
    todo.push_back(p);
  }
  if (todo.size() >= 2) {
    const size_t npx = size_t(w) * h;
    size_t lv = levels;
    for (size_t i = 0; i < todo.size(); ++i) lv = std::max(lv, todo[i]->requested_levels_);
    // One create call per role set (masks that also act in the current role need their own call), then ONE synchronisation
    // for the whole upload.  The staging vectors live until then.
    std::vector<RgbdImagePyramid*> groups[2];
    for (size_t i = 0; i < todo.size(); ++i) groups[!todo[i]->mask_.empty() && todo[i]->mask_current_ ? 1 : 0].push_back(todo[i]);
    std::vector<float> I[2], Z[2];
    std::vector<uint8_t> masks[2];   // per call: the pyramids without a mask get an all-usable one
    std::vector<dvo_b200_pyramid*> handles[2];
    const IntrinsicMatrix& k = todo[0]->camera_.level(0).intrinsics();
    for (int gi = 0; gi < 2; ++gi) {
      const std::vector<RgbdImagePyramid*>& g = groups[gi];
      const size_t n = g.size();
      if (n == 0) continue;
      I[gi].resize(n * npx); Z[gi].resize(n * npx);
      bool any_mask = false;
      for (size_t i = 0; i < n; ++i) {
        for (int y = 0; y < h; ++y) {   // row by row: a cv::Mat need not be continuous
          std::memcpy(&I[gi][i * npx + size_t(y) * w], g[i]->levels_[0]->intensity.ptr<float>(y), sizeof(float) * w);
          std::memcpy(&Z[gi][i * npx + size_t(y) * w], g[i]->levels_[0]->depth.ptr<float>(y), sizeof(float) * w);
        }
        any_mask = any_mask || !g[i]->mask_.empty();
      }
      if (any_mask)
        for (size_t i = 0; i < n; ++i) append_mask(g[i]->mask_, w, h, masks[gi]);
      handles[gi].resize(n);
      int rc = dvo_b200_pyramid_create_masked_batch_roles(ctx, int(n), DVO_B200_INPUT_FLOAT32, I[gi].data(), Z[gi].data(), 0.f,
                                                          any_mask ? masks[gi].data() : nullptr, mask_roles(gi == 1), w, h, k.fx(),
                                                          k.fy(), k.ox(), k.oy(), int(lv), handles[gi].data());
      if (rc != 0) throw std::runtime_error(std::string("dvo_b200_pyramid_create_masked_batch_roles: ") + dvo_b200_last_error(ctx));
    }
    dvo_b200_synchronize(ctx);   // one synchronisation for the whole upload: the staging vectors go out of scope
    for (int gi = 0; gi < 2; ++gi)
      for (size_t i = 0; i < groups[gi].size(); ++i) {
        RgbdImagePyramid* p = groups[gi][i];
        std::lock_guard<std::mutex> lock(p->mutex_);
        if (p->device_) dvo_b200_pyramid_release(p->device_);
        p->device_ = handles[gi][i];
        p->device_ctx_ = ctx;
        p->device_levels_ = lv;
      }
  }
  for (size_t i = 0; i < pyramids.size(); ++i) out[i] = pyramids[i]->device(ctx, levels);   // the rest one by one
}

RgbdImage& RgbdImagePyramid::level(size_t idx) {
  if (idx < levels_.size() && (idx == 0 || levels_[idx]->hasIntensity())) return *levels_[idx];
  if (!device_ || device_levels_ <= idx)
    throw std::runtime_error("RgbdImagePyramid::level: level not built (call build/compute and match first)");
  while (levels_.size() <= idx) levels_.push_back(camera_.level(levels_.size()).create());
  int w = 0, h = 0;
  float K[4];
  dvo_b200_pyramid_level_info(device_, int(idx), &w, &h, K);
  std::vector<float> planes(size_t(6) * w * h);
  // no context: the pyramid may be read after the tracker (and context) that uploaded it is gone
  if (dvo_b200_pyramid_download(nullptr, device_, int(idx), planes.data()) != 0)
    throw std::runtime_error("dvo_b200_pyramid_download failed");
  RgbdImage& img = *levels_[idx];
  cv::Mat* dst[6] = {&img.intensity, &img.depth, &img.intensity_dx, &img.intensity_dy, &img.depth_dx, &img.depth_dy};
  for (int c = 0; c < 6; ++c) {
    dst[c]->create(h, w, CV_32FC1);
    std::memcpy(dst[c]->ptr<float>(), planes.data() + size_t(c) * w * h, sizeof(float) * w * h);
  }
  return img;
}

}  // namespace core

// ---- DenseTracker -------------------------------------------------------------------------------------
DenseTracker::Config::Config()   // dense_tracking_config.cpp:27-42
    : FirstLevel(3), LastLevel(1), MaxIterationsPerLevel(100), Precision(5e-7), Mu(0), UseInitialEstimate(false),
      UseWeighting(true), UseParallel(false), InfluenceFuntionType(core::InfluenceFunctions::TDistribution),
      InfluenceFunctionParam(5.0f), ScaleEstimatorType(core::ScaleEstimators::TDistribution), ScaleEstimatorParam(5.0f),
      IntensityDerivativeThreshold(0.0f), DepthDerivativeThreshold(0.0f) {}

const DenseTracker::Config& DenseTracker::getDefaultConfig() {
  static Config c;
  return c;
}

DenseTracker::DenseTracker(const Config& config)
    : ctx_(0), collect_iterations_(false), corrected_estimator_(false), reference_selection_(selection_predicate_) { configure(config); }
DenseTracker::DenseTracker(const DenseTracker& other)
    : ctx_(0), collect_iterations_(other.collect_iterations_), corrected_estimator_(other.corrected_estimator_),
      reference_selection_(selection_predicate_) {
  configure(other.configuration());
}

void DenseTracker::useCorrectedEstimator(bool on) {
  corrected_estimator_ = on;
  if (ctx_) dvo_b200_set_estimator(ctx_, on ? DVO_B200_ESTIMATOR_CORRECTED : DVO_B200_ESTIMATOR_REFERENCE);
}
DenseTracker::~DenseTracker() {
  if (ctx_) dvo_b200_destroy(ctx_);
}

void DenseTracker::configure(const Config& config) {   // dense_tracking.cpp:72-97
  assert(config.IsSane());
  cfg = config;
  selection_predicate_.intensity_threshold = cfg.IntensityDerivativeThreshold;
  selection_predicate_.depth_threshold = cfg.DepthDerivativeThreshold;
}

dvo_b200_ctx* DenseTracker::context() {
  if (!ctx_) {
    const char* dev = std::getenv("DVO_B200_DEVICE");
    int rc = dvo_b200_create(dev ? std::atoi(dev) : 0, 0, &ctx_);
    if (rc != 0) throw std::runtime_error("dvo_b200_create failed: no usable CUDA device (the engine has no CPU fallback)");
    if (corrected_estimator_) dvo_b200_set_estimator(ctx_, DVO_B200_ESTIMATOR_CORRECTED);
  }
  return ctx_;
}

DenseTracker::Result::Result() : LogLikelihood(std::numeric_limits<double>::max()) {   // dense_tracking_config.cpp:101-108
  double nan = std::numeric_limits<double>::quiet_NaN();
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) Transformation.matrix()(i, j) = nan;
  Information.setIdentity();
}
bool DenseTracker::Result::isNaN() const {   // dense_tracking_config.cpp:96-99
  return !std::isfinite(Transformation.matrix().sum()) || !std::isfinite(Information.sum());
}
void DenseTracker::Result::setIdentity() {
  Transformation.setIdentity();
  Information.setIdentity();
  LogLikelihood = 0.0;
}

// dense_tracking_config.cpp:122-135.  EstimateInformation = A + mu*I is symmetric, so the real parts the reference takes from
// Eigen::EigenSolver are the eigenvalues of a symmetric matrix: cyclic Jacobi rotations on a copy, sorted ascending.
void DenseTracker::IterationStats::InformationEigenValues(core::Vector6d& eigenvalues) const {
  double a[6][6];
  for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) a[i][j] = 0.5 * (EstimateInformation(i, j) + EstimateInformation(j, i));
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < 6; ++i) { diag += a[i][i] * a[i][i]; for (int j = i + 1; j < 6; ++j) off += a[i][j] * a[i][j]; }
    if (!(off > 1e-32 * diag)) break;
    for (int p = 0; p < 5; ++p)
      for (int q = p + 1; q < 6; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double cs = 1.0 / std::sqrt(t * t + 1.0), sn = t * cs;
        for (int k = 0; k < 6; ++k) { const double x = a[k][p], y = a[k][q]; a[k][p] = cs * x - sn * y; a[k][q] = sn * x + cs * y; }
        for (int k = 0; k < 6; ++k) { const double x = a[p][k], y = a[q][k]; a[p][k] = cs * x - sn * y; a[q][k] = sn * x + cs * y; }
      }
  }
  double ev[6];
  for (int i = 0; i < 6; ++i) ev[i] = a[i][i];
  std::sort(ev, ev + 6);
  for (int i = 0; i < 6; ++i) eigenvalues(i) = ev[i];
}

double DenseTracker::IterationStats::InformationConditionNumber() const {
  core::Vector6d ev;
  InformationEigenValues(ev);
  return std::abs(ev(5) / ev(0));
}

bool DenseTracker::LevelStats::HasIterationWithIncrement() const {   // dense_tracking_config.cpp:138-143
  int min = TerminationCriterion == TerminationCriteria::LogLikelihoodDecreased || TerminationCriterion == TerminationCriteria::TooFewConstraints ? 2 : 1;
  return int(Iterations.size()) >= min;
}
DenseTracker::IterationStats& DenseTracker::LevelStats::LastIterationWithIncrement() {
  assert(HasIterationWithIncrement());
  return TerminationCriterion == TerminationCriteria::LogLikelihoodDecreased ? Iterations[Iterations.size() - 2] : Iterations[Iterations.size() - 1];
}
const DenseTracker::IterationStats& DenseTracker::LevelStats::LastIterationWithIncrement() const {
  assert(HasIterationWithIncrement());
  return TerminationCriterion == TerminationCriteria::LogLikelihoodDecreased ? Iterations[Iterations.size() - 2] : Iterations[Iterations.size() - 1];
}

bool DenseTracker::match(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current, core::AffineTransformd& transformation) {
  Result result;
  result.Transformation = transformation;
  bool ok = match(reference, current, result);
  transformation = result.Transformation;
  return ok;
}
bool DenseTracker::match(core::PointSelection& reference, core::RgbdImagePyramid& current, core::AffineTransformd& transformation) {
  Result result;
  result.Transformation = transformation;
  bool ok = match(reference, current, result);
  transformation = result.Transformation;
  return ok;
}
bool DenseTracker::match(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current, Result& result) {   // dense_tracking.cpp:123-129
  reference.compute(cfg.getNumLevels());
  reference_selection_.setRgbdImagePyramid(reference);
  return match(reference_selection_, current, result);
}
bool DenseTracker::match(core::PointSelection& reference, core::RgbdImagePyramid& current, Result& result) {
  std::vector<core::RgbdImagePyramid*> refs(1, &reference.getRgbdImagePyramid()), curs(1, &current);
  std::vector<Result> results(1, result);
  bool ok = matchBatch(refs, curs, results);
  result = results[0];
  return ok;
}

static void fill_result(const dvo_b200_result& r, const dvo_b200_iteration_stats* its, DenseTracker::Result& out) {
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) out.Transformation.matrix()(i, j) = r.transformation[i * 4 + j];
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) out.Information(i, j) = r.information[i * 6 + j];
  out.LogLikelihood = r.log_likelihood;
  int cursor = 0;
  for (int l = 0; l < r.num_levels; ++l) {   // match() appends to Statistics.Levels (dense_tracking.cpp:202)
    const dvo_b200_level_stats& ls = r.levels[l];
    DenseTracker::LevelStats s;
    s.Id = size_t(ls.id); s.MaxValidPixels = size_t(ls.max_valid_pixels); s.ValidPixels = size_t(ls.valid_pixels);
    s.TerminationCriterion = DenseTracker::TerminationCriteria::Enum(ls.termination);
    s.Iterations.resize(size_t(ls.num_iterations));
    for (int k = 0; k < ls.num_iterations; ++k) {
      DenseTracker::IterationStats& it = s.Iterations[size_t(k)];
      it.Id = size_t(k); it.ValidConstraints = 0; it.TDistributionLogLikelihood = 0; it.PriorLogLikelihood = 0;
      if (its) {
        const dvo_b200_iteration_stats& q = its[cursor + k];
        it.ValidConstraints = size_t(q.valid_constraints);
        it.TDistributionLogLikelihood = q.tdist_log_likelihood;
        it.PriorLogLikelihood = q.prior_log_likelihood;
        for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) it.TDistributionPrecision(a, b) = q.tdist_precision[a * 2 + b];
        for (int a = 0; a < 6; ++a) it.EstimateIncrement(a) = q.increment[a];
        for (int a = 0; a < 6; ++a) for (int b = 0; b < 6; ++b) it.EstimateInformation(a, b) = q.information[a * 6 + b];
      }
    }
    // without the optional per-iteration log the fields the callers read are still filled
    // (keyframe_tracker.cpp:167, constraint_proposal_voter.cpp:128-129)
    if (!its && ls.num_iterations > 0) {
      s.Iterations.back().ValidConstraints = size_t(ls.last_valid_constraints);
      if (ls.has_iteration_with_increment) {
        DenseTracker::IterationStats& li = s.LastIterationWithIncrement();
        li.ValidConstraints = size_t(ls.last_increment_valid_constraints);
        li.TDistributionLogLikelihood = ls.last_increment_log_likelihood;
      }
    }
    cursor += ls.num_iterations;
    out.Statistics.Levels.push_back(s);
  }
}

// the dvo_b200_config of a DenseTracker::Config
static dvo_b200_config b200_config(const DenseTracker::Config& cfg, bool use_initial_estimate) {
  dvo_b200_config c;
  dvo_b200_config_default(&c);
  c.first_level = cfg.FirstLevel; c.last_level = cfg.LastLevel; c.max_iterations_per_level = cfg.MaxIterationsPerLevel;
  c.use_initial_estimate = use_initial_estimate ? 1 : 0; c.precision = cfg.Precision; c.mu = cfg.Mu;
  c.intensity_derivative_threshold = cfg.IntensityDerivativeThreshold; c.depth_derivative_threshold = cfg.DepthDerivativeThreshold;
  return c;
}

// entries of the per-iteration log per pair, 0 without one
static int iteration_log_size(const DenseTracker::Config& c, bool on) { return on ? (c.FirstLevel - c.LastLevel + 1) * (c.MaxIterationsPerLevel + 1) : 0; }

// device mirrors of n reference pyramids, then of n current pyramids: one upload, one synchronisation
static std::vector<dvo_b200_pyramid*> upload_pairs(dvo_b200_ctx* ctx, const DenseTracker::Config& cfg,
                                                   const std::vector<core::RgbdImagePyramid*>& references,
                                                   const std::vector<core::RgbdImagePyramid*>& currents) {
  std::vector<core::RgbdImagePyramid*> all(references);
  all.insert(all.end(), currents.begin(), currents.end());
  for (size_t i = 0; i < all.size(); ++i) all[i]->compute(cfg.getNumLevels());   // dense_tracking.cpp:133
  std::vector<dvo_b200_pyramid*> dev;
  core::RgbdImagePyramid::deviceBatch(ctx, all, cfg.getNumLevels(), dev);
  return dev;
}

// the weight map of one alignment at last_level, in host memory, written straight into the cv::Mat
static dvo_b200_weight_maps host_weight_map(dvo_b200_pyramid* reference, int last_level, cv::Mat& weights) {
  int w = 0, h = 0;
  dvo_b200_pyramid_level_info(reference, last_level, &w, &h, 0);
  weights.create(h, w, CV_32FC1);
  dvo_b200_weight_maps maps;
  std::memset(&maps, 0, sizeof(maps));
  maps.memory = DVO_B200_MAPS_HOST;
  maps.weight.data = weights.ptr<float>();
  maps.weight.row_bytes = int64_t(sizeof(float)) * w;
  maps.weight.image_bytes = maps.weight.row_bytes * h;
  return maps;
}

// n R x R matrices, matrix(j) for j < n, as row-major doubles: matrix j at R * R * j
template <int R, class F>
static std::vector<double> row_major(size_t n, F matrix) {
  std::vector<double> v(R * R * n);
  for (size_t j = 0; j < n; ++j)
    for (int a = 0; a < R; ++a)
      for (int b = 0; b < R; ++b) v[R * R * j + a * R + b] = matrix(j)(a, b);
  return v;
}

bool DenseTracker::matchBatch(const std::vector<core::RgbdImagePyramid*>& references, const std::vector<core::RgbdImagePyramid*>& currents,
                              std::vector<Result>& results) {
  return matchBatch(references, currents, static_cast<const double*>(0), results);
}

bool DenseTracker::matchWithPrior(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current,
                                  const core::Matrix6d& prior_information, Result& result) {
  std::vector<core::RgbdImagePyramid*> refs(1, &reference), curs(1, &current);
  std::vector<core::Matrix6d> priors(1, prior_information);
  std::vector<Result> results(1, result);
  const bool ok = matchBatch(refs, curs, priors, results);
  if (ok) result = results[0];
  return ok;
}

bool DenseTracker::matchBatch(const std::vector<core::RgbdImagePyramid*>& references, const std::vector<core::RgbdImagePyramid*>& currents,
                              const std::vector<core::Matrix6d>& prior_information, std::vector<Result>& results) {
  const size_t n = references.size();
  if (prior_information.size() != n) return false;
  const std::vector<double> L = row_major<6>(n, [&](size_t i) { return prior_information[i]; });
  std::vector<Result> out(results);
  out.resize(n);
  if (!matchBatch(references, currents, n ? L.data() : 0, out)) return false;
  results = out;
  return true;
}

bool DenseTracker::matchWithWeights(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current, Result& result,
                                    cv::Mat& weights) {
  std::vector<core::RgbdImagePyramid*> refs(1, &reference), curs(1, &current);
  std::vector<Result> results(1, result);
  const bool ok = matchBatch(refs, curs, static_cast<const double*>(0), results, &weights);
  if (ok) result = results[0];
  return ok;
}

bool DenseTracker::matchWithHypotheses(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current,
                                       const std::vector<core::AffineTransformd>& initial, int screen_level, Result& result, int* best,
                                       double min_constraint_ratio) {
  return matchWithHypotheses(reference, current, initial, static_cast<const double*>(0), screen_level, result, best, min_constraint_ratio, 0);
}

bool DenseTracker::matchWithHypotheses(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current,
                                       const std::vector<core::AffineTransformd>& initial, const std::vector<core::Matrix6d>& prior_information,
                                       int screen_level, Result& result, int* best, double min_constraint_ratio, cv::Mat* weights) {
  if (prior_information.size() != initial.size()) return false;
  const std::vector<double> L = row_major<6>(initial.size(), [&](size_t j) { return prior_information[j]; });
  return matchWithHypotheses(reference, current, initial, L.data(), screen_level, result, best, min_constraint_ratio, weights);
}

// Both public forms: prior (k * 36, Lambda of hypothesis j at 36 j) or NULL, and the weight map of the continued alignment at
// LastLevel, in host memory, if weights is given.
bool DenseTracker::matchWithHypotheses(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current,
                                       const std::vector<core::AffineTransformd>& initial, const double* prior, int screen_level,
                                       Result& result, int* best, double min_constraint_ratio, cv::Mat* weights) {
  dvo_b200_config c = b200_config(cfg, true);
  const int k = int(initial.size());
  std::vector<double> H = row_major<4>(initial.size(), [&](size_t j) { return initial[j].matrix(); });
  dvo_b200_result raw;
  int32_t chosen = 0;
  if (!dvo_b200::hypotheses_args_error(&c, 1, k, H.data(), screen_level, min_constraint_ratio, &raw, &chosen).empty()) return false;
  if (prior) {   // the prior checks of dvo_b200_match_batch_hypotheses_modes, refused before any upload
    if (c.mu != 0.0) return false;
    for (int j = 0; j < k; ++j)
      if (!dvo_b200::prior_matrix_error(prior + 36 * (size_t)j).empty()) return false;
  }
  dvo_b200_ctx* ctx = context();
  std::vector<dvo_b200_pyramid*> dev = upload_pairs(ctx, cfg, {&reference}, {&current});
  const int max_log = iteration_log_size(cfg, collect_iterations_);
  std::vector<dvo_b200_iteration_stats> its((size_t)max_log);
  dvo_b200_weight_maps maps;
  if (weights) maps = host_weight_map(dev[0], c.last_level, *weights);   // of the continued alignment
  if (dvo_b200_match_batch_hypotheses_modes(ctx, &c, 1, &dev[0], &dev[1], k, H.data(), screen_level, min_constraint_ratio, prior, 0, 0, 0,
                                            &raw, &chosen, 0, 0, max_log ? its.data() : 0, max_log, weights ? &maps : 0) != 0)
    throw std::runtime_error(std::string("dvo_b200_match_batch_hypotheses_modes: ") + dvo_b200_last_error(ctx));
  Result out;
  fill_result(raw, max_log ? its.data() : 0, out);
  result = out;
  if (best) *best = chosen;
  return true;
}

bool DenseTracker::matchBatch(const std::vector<core::RgbdImagePyramid*>& references, const std::vector<core::RgbdImagePyramid*>& currents,
                              const double* prior_information, std::vector<Result>& results, cv::Mat* weights) {
  const size_t n = references.size();
  if (n == 0 || currents.size() != n) return false;
  if (prior_information) {   // refused before any upload
    dvo_b200_config pc;
    pc.mu = cfg.Mu;
    if (!dvo_b200::prior_args_error(&pc, int(n), prior_information, 0, 0).empty()) return false;
  }
  results.resize(n);
  dvo_b200_ctx* ctx = context();
  const dvo_b200_config c = b200_config(cfg, cfg.UseInitialEstimate);
  std::vector<dvo_b200_pyramid*> dev = upload_pairs(ctx, cfg, references, currents);
  for (size_t i = 0; i < n; ++i)
    if (cfg.UseInitialEstimate) assert(!results[i].isNaN() && "Provided initialization is NaN!");
  const std::vector<double> T = row_major<4>(n, [&](size_t i) { return results[i].Transformation.matrix(); });
  std::vector<dvo_b200_result> raw(n);
  const int max_log = iteration_log_size(cfg, collect_iterations_);
  std::vector<dvo_b200_iteration_stats> log(size_t(max_log) * n);
  const double* T0 = cfg.UseInitialEstimate ? T.data() : 0;
  int rc;
  if (weights) {   // of the one pair
    dvo_b200_weight_maps maps = host_weight_map(dev[0], c.last_level, *weights);
    rc = dvo_b200_match_batch_maps(ctx, &c, int(n), &dev[0], &dev[n], T0, 0, 0, 0, raw.data(), max_log ? log.data() : 0, max_log,
                                   &maps);
  } else if (prior_information) {
    rc = dvo_b200_match_batch_prior(ctx, &c, int(n), &dev[0], &dev[n], T0, prior_information, 0, 0, raw.data(),
                                    max_log ? log.data() : 0, max_log);
  } else {
    rc = dvo_b200_match_batch(ctx, &c, int(n), &dev[0], &dev[n], T0, raw.data(), max_log ? log.data() : 0, max_log);
  }
  if (rc != 0) throw std::runtime_error(std::string("dvo_b200_match_batch: ") + dvo_b200_last_error(ctx));
  for (size_t i = 0; i < n; ++i) fill_result(raw[i], max_log ? &log[size_t(max_log) * i] : 0, results[i]);
  return true;   // the reference's match() always returns true (dense_tracking.cpp:135,375)
}

cv::Mat DenseTracker::computeIntensityErrorImage(core::RgbdImagePyramid& reference, core::RgbdImagePyramid& current,
                                                 const core::AffineTransformd& transformation, size_t level) {
  dvo_b200_ctx* ctx = context();
  reference.compute(level + 1);
  current.compute(level + 1);
  dvo_b200_pyramid* r = reference.device(ctx, level + 1);
  dvo_b200_pyramid* q = current.device(ctx, level + 1);
  int w = 0, h = 0;
  float K[4];
  dvo_b200_pyramid_level_info(r, int(level), &w, &h, K);
  double T[16];
  for (int a = 0; a < 4; ++a) for (int b = 0; b < 4; ++b) T[a * 4 + b] = transformation.matrix()(a, b);
  dvo_b200_config c;
  dvo_b200_config_default(&c);
  c.intensity_derivative_threshold = cfg.IntensityDerivativeThreshold; c.depth_derivative_threshold = cfg.DepthDerivativeThreshold;
  cv::Mat result = cv::Mat::zeros(h, w, CV_32FC1);
  if (dvo_b200_intensity_error_image(ctx, &c, r, q, int(level), T, result.ptr<float>(), nullptr) != 0)
    throw std::runtime_error(std::string("dvo_b200_intensity_error_image: ") + dvo_b200_last_error(ctx));
  return result;
}

}  // namespace dvo

std::ostream& operator<<(std::ostream& out, const dvo::DenseTracker::Config& c) {
  return out << "First Level = " << c.FirstLevel << ", Last Level = " << c.LastLevel << ", Max Iterations per Level = " << c.MaxIterationsPerLevel
             << ", Precision = " << c.Precision << ", Mu = " << c.Mu << ", Use Initial Estimate = " << (c.UseInitialEstimate ? "true" : "false")
             << ", Use Weighting = " << (c.UseWeighting ? "true" : "false") << ", Intensity Derivative Threshold = " << c.IntensityDerivativeThreshold
             << ", Depth Derivative Threshold = " << c.DepthDerivativeThreshold;
}
std::ostream& operator<<(std::ostream& o, const dvo::DenseTracker::IterationStats& s) {
  return o << "Iteration: " << s.Id << " ValidConstraints: " << s.ValidConstraints << " DataLogLikelihood: " << s.TDistributionLogLikelihood
           << " PriorLogLikelihood: " << s.PriorLogLikelihood << std::endl;
}
std::ostream& operator<<(std::ostream& o, const dvo::DenseTracker::LevelStats& s) {
  static const char* names[] = {"IterationsExceeded", "IncrementTooSmall", "LogLikelihoodDecreased", "TooFewConstraints"};
  int t = int(s.TerminationCriterion);
  o << "Level: " << s.Id << " Pixel: " << s.ValidPixels << "/" << s.MaxValidPixels << " Termination: " << (t >= 0 && t < 4 ? names[t] : "")
    << " Iterations: " << s.Iterations.size() << std::endl;
  for (size_t i = 0; i < s.Iterations.size(); ++i) o << s.Iterations[i];
  return o;
}
std::ostream& operator<<(std::ostream& o, const dvo::DenseTracker::Stats& s) {
  o << s.Levels.size() << " levels" << std::endl;
  for (size_t i = 0; i < s.Levels.size(); ++i) o << s.Levels[i];
  return o;
}
