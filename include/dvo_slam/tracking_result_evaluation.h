// dvo_slam/tracking_result_evaluation.h -- the keyframe-selection scores dvo_slam computes from DenseTracker
// results (reference interface: dvo_slam/include/dvo_slam/tracking_result_evaluation.h:31-80, behaviour:
// dvo_slam/src/tracking_result_evaluation.cpp:26-62).  They read only Result fields the CUDA engine fills
// (Information, LogLikelihood, the last iteration's ValidConstraints), so they sit on the adapter unchanged:
// same class names, constructors and virtuals; header-only here.
#ifndef DVO_SLAM_TRACKING_RESULT_EVALUATION_H_
#define DVO_SLAM_TRACKING_RESULT_EVALUATION_H_

#include <cmath>

#include "dvo/dense_tracking.h"

namespace dvo_slam {

class TrackingResultEvaluation {
 public:
  typedef dvo_b200::compat::shared_ptr<TrackingResultEvaluation> Ptr;
  typedef dvo_b200::compat::shared_ptr<const TrackingResultEvaluation> ConstPtr;

  virtual ~TrackingResultEvaluation() {}

  // running sum of the score over the frames tracked against the current keyframe (tracking_result_evaluation.cpp:26-30)
  virtual void add(const dvo::DenseTracker::Result& r) { sum_ += value(r); count_ += 1.0; }
  // score of r relative to the first frame after the keyframe (:32-35)
  virtual double ratioWithFirst(const dvo::DenseTracker::Result& r) const { return value(r) / first_; }
  // score of r relative to the mean so far (:37-40)
  virtual double ratioWithAverage(const dvo::DenseTracker::Result& r) const { return value(r) / sum_ * count_; }

 protected:
  explicit TrackingResultEvaluation(double first) : first_(first), sum_(first), count_(1.0) {}
  virtual double value(const dvo::DenseTracker::Result& r) const = 0;

 private:
  double first_, sum_, count_;
};

// -LogLikelihood (:54-57)
class LogLikelihoodTrackingResultEvaluation : public TrackingResultEvaluation {
 public:
  explicit LogLikelihoodTrackingResultEvaluation(const dvo::DenseTracker::Result& r) : TrackingResultEvaluation(score(r)) {}
  virtual double value(const dvo::DenseTracker::Result& r) const { return score(r); }
 private:
  static double score(const dvo::DenseTracker::Result& r) { return -r.LogLikelihood; }
};

// -LogLikelihood per constraint of the last iteration on the finest level (:59-62)
class NormalizedLogLikelihoodTrackingResultEvaluation : public TrackingResultEvaluation {
 public:
  explicit NormalizedLogLikelihoodTrackingResultEvaluation(const dvo::DenseTracker::Result& r) : TrackingResultEvaluation(score(r)) {}
  virtual double value(const dvo::DenseTracker::Result& r) const { return score(r); }
 private:
  static double score(const dvo::DenseTracker::Result& r) {
    return -r.LogLikelihood / double(r.Statistics.Levels.back().Iterations.back().ValidConstraints);
  }
};

// log det(Information): the entropy-ratio keyframe criterion (:49-52)
class EntropyRatioTrackingResultEvaluation : public TrackingResultEvaluation {
 public:
  explicit EntropyRatioTrackingResultEvaluation(const dvo::DenseTracker::Result& r) : TrackingResultEvaluation(score(r)) {}
  virtual double value(const dvo::DenseTracker::Result& r) const { return score(r); }
 private:
  static double score(const dvo::DenseTracker::Result& r) { return std::log(r.Information.determinant()); }
};

}  // namespace dvo_slam

#endif
