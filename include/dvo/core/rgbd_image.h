// dvo/core/rgbd_image.h -- adapter counterpart of dvo_core/include/dvo/core/rgbd_image.h:94-262.
// Same class names and member functions for the part of the image model that DenseTracker::match()
// and its callers use; the pixels live in a device pyramid (dvo_b200_pyramid) that is created lazily
// and shared by every tracker that aligns against this image.
#ifndef DVO_B200_ADAPTER_RGBD_IMAGE_H_
#define DVO_B200_ADAPTER_RGBD_IMAGE_H_
#include <cstddef>
#include <mutex>
#include <vector>
#include "../../dvo_b200.h"
#include "datatypes.h"
#include "intrinsic_matrix.h"

namespace dvo { namespace core {

class RgbdImage;
class RgbdImagePyramid;
class RgbdCameraPyramid;
typedef dvo_b200::compat::shared_ptr<RgbdImage> RgbdImagePtr;
typedef dvo_b200::compat::shared_ptr<RgbdImagePyramid> RgbdImagePyramidPtr;

class RgbdCamera {   // rgbd_image.h:99-122
 public:
  RgbdCamera(size_t width, size_t height, const IntrinsicMatrix& intrinsics) : width_(width), height_(height), intrinsics_(intrinsics) {}
  size_t width() const { return width_; }
  size_t height() const { return height_; }
  const IntrinsicMatrix& intrinsics() const { return intrinsics_; }
  RgbdImagePtr create(const cv::Mat& intensity, const cv::Mat& depth) const;
  RgbdImagePtr create() const;
 private:
  size_t width_, height_;
  IntrinsicMatrix intrinsics_;
};
typedef dvo_b200::compat::shared_ptr<RgbdCamera> RgbdCameraPtr;

class RgbdCameraPyramid {   // rgbd_image.h:127-144
 public:
  RgbdCameraPyramid(const RgbdCamera& base);
  RgbdCameraPyramid(size_t base_width, size_t base_height, const IntrinsicMatrix& base_intrinsics);
  RgbdImagePyramidPtr create(const cv::Mat& base_intensity, const cv::Mat& base_depth);
  void build(size_t levels);
  const RgbdCamera& level(size_t level);
  const RgbdCamera& level(size_t level) const;
 private:
  std::vector<RgbdCameraPtr> levels_;
};

class RgbdImage {   // rgbd_image.h:150-236 (public data members kept; warp*/normals helpers are not on the hot path)
 public:
  explicit RgbdImage(const RgbdCamera& camera) : width(camera.width()), height(camera.height()), timestamp(0), camera_(camera) {}
  const RgbdCamera& camera() const { return camera_; }
  cv::Mat intensity, intensity_dx, intensity_dy, depth, depth_dx, depth_dy, rgb;
  size_t width, height;
  double timestamp;
  bool hasIntensity() const { return !intensity.empty(); }
  bool hasDepth() const { return !depth.empty(); }
  bool hasRgb() const { return !rgb.empty(); }
  void initialize() { width = camera_.width(); height = camera_.height(); }
  void calculateDerivatives() {}          // derivatives are built on the device with the pyramid
  void buildPointCloud() {}
  void buildAccelerationStructure() {}
  bool inImage(const float& x, const float& y) const { return x >= 0 && x < width && y >= 0 && y < height; }
 private:
  const RgbdCamera& camera_;
};

class RgbdImagePyramid {   // rgbd_image.h:242-262
 public:
  RgbdImagePyramid(RgbdCameraPyramid& camera, const cv::Mat& intensity, const cv::Mat& depth);
  virtual ~RgbdImagePyramid();
  void compute(const size_t num_levels) { build(num_levels); }
  void build(const size_t num_levels);
  RgbdImage& level(size_t idx);
  double timestamp() const;

  // --- extension used by the adapter's DenseTracker: the device mirror with at least `levels` levels,
  // created on first use through `ctx` (uploads level 0 and builds the pyramid on the GPU). ---
  dvo_b200_pyramid* device(dvo_b200_ctx* ctx, size_t levels);
  // the same for many pyramids at once: every pyramid that still needs its device mirror is uploaded in ONE
  // dvo_b200_pyramid_create_batch call followed by ONE synchronisation (pyramids that appear several times in the
  // list -- a keyframe in several proposals -- are uploaded once); out[i] = device mirror of pyramids[i]
  static void deviceBatch(dvo_b200_ctx* ctx, const std::vector<RgbdImagePyramid*>& pyramids, size_t levels,
                          std::vector<dvo_b200_pyramid*>& out);
  // --- extension: a reference mask, CV_8U of the base size, nonzero = usable, 0 = excluded.  Excluded pixels never become
  // constraints while this pyramid is the reference of an alignment, at any level (a coarse pixel is usable iff its whole
  // footprint is; dvo_b200_pyramid_create_masked_batch).  The mask is copied.  Returns false and changes nothing once the
  // device mirror exists (after the first match) or if the size or type is wrong. ---
  bool setReferenceMask(const cv::Mat& mask);
  // --- extension: the same mask, and with current_role_too also in the current role: while this pyramid is the current
  // image of an alignment, a warped point is rejected iff one of its four bilinear taps is unusable at that level
  // (dvo_b200_pyramid_create_masked_batch_roles).  The same rules as setReferenceMask, which is setMask(mask, false). ---
  bool setMask(const cv::Mat& mask, bool current_role_too);
 private:
  RgbdCameraPyramid& camera_;
  std::vector<RgbdImagePtr> levels_;
  cv::Mat mask_;   // setMask; empty: no mask
  bool mask_current_;   // setMask(mask, true): the mask also acts in the current role
  dvo_b200_pyramid* device_;
  dvo_b200_ctx* device_ctx_;
  size_t device_levels_, requested_levels_;
  std::mutex mutex_;
};

} }
#endif
