// tum_replay.cpp -- TUM RGB-D sequence replay without ROS (SURVEY.md 8f row N3).
//
// What it mirrors from dvo_benchmark:
//   * association / ground-truth readers: `ts rgb_file ts depth_file` and `ts tx ty tz qx qy qz qw` lines, '#'
//     comments skipped (dvo_benchmark/include/dvo_benchmark/file_reader.h:35-113, rgbd_pair.h:59-71,
//     groundtruth.h:65-79), first pose = the ground-truth entry closest after the first RGB stamp
//     (tools.h:68-82, benchmark_slam.cpp:421-429);
//   * the loader: 8-bit colour -> grey -> float32, 16-bit depth * 1/5000 with 0 -> NaN (benchmark_slam.cpp:45-93);
//   * the frame-to-frame odometry loop and the trajectory file: match(reference, current, relative);
//     trajectory = trajectory * relative; one line `ts tx ty tz qx qy qz qw ` per frame
//     (dvo_benchmark/src/benchmark.cpp:407-480, benchmark_slam.cpp:494-503).
// What is new: consecutive pairs do not depend on each other, so they are aligned `--batch` at a time with
// DenseTracker::matchBatch; the trajectory is accumulated afterwards.  The keyframe graph of benchmark_slam is
// out of scope (SURVEY.md 8).
//
// PNG decoding (the TUM file format) uses zlib only: non-interlaced 8-bit grey / RGB / RGBA and 16-bit grey.
#include <zlib.h>

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "dvo/dense_tracking.h"

namespace {

struct RgbdPair { double rgb_stamp, depth_stamp; std::string rgb_file, depth_file; };
struct Groundtruth { double stamp, p[3], q[4]; };   // q = x y z w

std::istream& operator>>(std::istream& in, RgbdPair& e) { return in >> e.rgb_stamp >> e.rgb_file >> e.depth_stamp >> e.depth_file; }
std::istream& operator>>(std::istream& in, Groundtruth& e) {
  return in >> e.stamp >> e.p[0] >> e.p[1] >> e.p[2] >> e.q[0] >> e.q[1] >> e.q[2] >> e.q[3];
}

template <class Entry>
bool read_entries(const std::string& path, std::vector<Entry>& out) {
  std::ifstream f(path.c_str());
  if (!f) return false;
  std::string line;
  while (std::getline(f, line)) {
    size_t a = line.find_first_not_of(" \t\r");
    if (a == std::string::npos || line[a] == '#') continue;     // FileReader::skipComments
    std::istringstream ls(line);
    Entry e;
    if (ls >> e) out.push_back(e);
  }
  return true;
}

// ros::Time prints sec.nsec with nine digits; ros::Time::fromSec splits a double the same way
std::string stamp_text(double t) {
  long long sec = (long long)std::floor(t);
  long long nsec = (long long)std::llround((t - (double)sec) * 1e9);
  if (nsec >= 1000000000LL) { sec += 1; nsec -= 1000000000LL; }
  char buf[64];
  std::snprintf(buf, sizeof buf, "%lld.%09lld", sec, nsec);
  return buf;
}

// ---- PNG ------------------------------------------------------------------------------------------------
struct Image { int w = 0, h = 0, channels = 0, bits = 0; std::vector<uint16_t> px; };   // interleaved channels

uint32_t be32(const unsigned char* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }

bool load_png(const std::string& path, Image& img, std::string& why) {
  std::ifstream f(path.c_str(), std::ios::binary);
  if (!f) { why = "cannot open " + path; return false; }
  std::vector<unsigned char> file((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
  static const unsigned char sig[8] = {0x89, 'P', 'N', 'G', 0x0d, 0x0a, 0x1a, 0x0a};
  if (file.size() < 8 || std::memcmp(file.data(), sig, 8) != 0) { why = "not a PNG: " + path; return false; }
  std::vector<unsigned char> idat;
  int color = -1, interlace = 0;
  for (size_t pos = 8; pos + 12 <= file.size();) {
    const uint32_t len = be32(&file[pos]);
    const char* type = reinterpret_cast<const char*>(&file[pos + 4]);
    if (pos + 12 + len > file.size()) { why = "truncated PNG: " + path; return false; }
    const unsigned char* data = &file[pos + 8];
    if (!std::memcmp(type, "IHDR", 4) && len >= 13) {
      img.w = int(be32(data)); img.h = int(be32(data + 4)); img.bits = data[8]; color = data[9]; interlace = data[12];
    } else if (!std::memcmp(type, "IDAT", 4)) {
      idat.insert(idat.end(), data, data + len);
    } else if (!std::memcmp(type, "IEND", 4)) {
      break;
    }
    pos += 12 + size_t(len);
  }
  img.channels = color == 0 ? 1 : color == 2 ? 3 : color == 4 ? 2 : color == 6 ? 4 : 0;
  if (!img.channels || interlace != 0 || !(img.bits == 8 || img.bits == 16) || img.w <= 0 || img.h <= 0) {
    why = "unsupported PNG flavour (need non-interlaced 8/16-bit grey, RGB or RGBA): " + path;
    return false;
  }
  const size_t bpp = size_t(img.channels) * img.bits / 8, stride = bpp * img.w;
  std::vector<unsigned char> raw((stride + 1) * img.h);
  uLongf raw_len = raw.size();
  if (uncompress(raw.data(), &raw_len, idat.data(), idat.size()) != Z_OK || raw_len != raw.size()) { why = "zlib: bad image data in " + path; return false; }
  std::vector<unsigned char> cur(stride), prev(stride, 0);
  img.px.resize(size_t(img.w) * img.h * img.channels);
  for (int y = 0; y < img.h; ++y) {
    const unsigned char* line = &raw[(stride + 1) * y];
    const int filter = line[0];
    for (size_t i = 0; i < stride; ++i) {
      const int a = i >= bpp ? cur[i - bpp] : 0, b = prev[i], c = i >= bpp ? prev[i - bpp] : 0;
      int pred = 0;
      switch (filter) {
        case 0: pred = 0; break;
        case 1: pred = a; break;
        case 2: pred = b; break;
        case 3: pred = (a + b) >> 1; break;
        case 4: { const int p = a + b - c, pa = std::abs(p - a), pb = std::abs(p - b), pc = std::abs(p - c); pred = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c); break; }
        default: why = "bad PNG filter in " + path; return false;
      }
      cur[i] = (unsigned char)(line[1 + i] + pred);
    }
    uint16_t* dst = &img.px[size_t(y) * img.w * img.channels];
    for (size_t i = 0; i < size_t(img.w) * img.channels; ++i)
      dst[i] = img.bits == 8 ? cur[i] : uint16_t((cur[2 * i] << 8) | cur[2 * i + 1]);     // PNG is big endian
    prev.swap(cur);
  }
  return true;
}

// the loader of benchmark_slam.cpp:45-93 on decoded images
bool to_grey_f32(const Image& rgb, cv::Mat& out, std::string& why) {
  if (rgb.bits != 8) { why = "colour image must be 8 bit"; return false; }
  out.create(rgb.h, rgb.w, CV_32FC1);
  float* o = out.ptr<float>();
  const size_t n = size_t(rgb.w) * rgb.h;
  if (rgb.channels == 1) {
    for (size_t i = 0; i < n; ++i) o[i] = float(rgb.px[i]);
  } else if (rgb.channels >= 3) {
    // cv::cvtColor(CV_BGR2GRAY) on 8-bit data is fixed point: (B*1868 + G*9617 + R*4899 + (1 << 13)) >> 14; PNG stores R,G,B
    for (size_t i = 0; i < n; ++i) {
      const int r = rgb.px[i * rgb.channels], g = rgb.px[i * rgb.channels + 1], b = rgb.px[i * rgb.channels + 2];
      o[i] = float((b * 1868 + g * 9617 + r * 4899 + (1 << 13)) >> 14);
    }
  } else { why = "colour image has an unsupported channel count"; return false; }
  return true;
}
bool to_depth_f32(const Image& d, float scale, cv::Mat& out, std::string& why) {
  if (d.channels != 1 || d.bits != 16) { why = "depth image must be 16-bit single channel"; return false; }
  out.create(d.h, d.w, CV_32FC1);
  float* o = out.ptr<float>();
  const float nan = std::numeric_limits<float>::quiet_NaN();
  for (size_t i = 0; i < size_t(d.w) * d.h; ++i) o[i] = d.px[i] == 0 ? nan : float(d.px[i]) * scale;   // surface_pyramid.cpp:65-105
  return true;
}

// ---- poses ----------------------------------------------------------------------------------------------
dvo::core::AffineTransformd pose_from(const Groundtruth& g) {
  dvo::core::AffineTransformd T;
  const double x = g.q[0], y = g.q[1], z = g.q[2], w = g.q[3];
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                       2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                       2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)};
  for (int i = 0; i < 3; ++i) { for (int j = 0; j < 3; ++j) T.matrix()(i, j) = R[3 * i + j]; T.matrix()(i, 3) = g.p[i]; }
  return T;
}
// rotation matrix -> unit quaternion (x y z w), the branch structure of Eigen::Quaterniond(Matrix3d)
void quaternion_of(const dvo::core::AffineTransformd& T, double q[4]) {
  double m[3][3];
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) m[i][j] = T.matrix()(i, j);
  double t = m[0][0] + m[1][1] + m[2][2];
  if (t > 0) {
    t = std::sqrt(t + 1.0);
    q[3] = 0.5 * t; t = 0.5 / t;
    q[0] = (m[2][1] - m[1][2]) * t; q[1] = (m[0][2] - m[2][0]) * t; q[2] = (m[1][0] - m[0][1]) * t;
  } else {
    int i = 0;
    if (m[1][1] > m[0][0]) i = 1;
    if (m[2][2] > m[i][i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m[i][i] - m[j][j] - m[k][k] + 1.0);
    q[i] = 0.5 * t; t = 0.5 / t;
    q[3] = (m[k][j] - m[j][k]) * t; q[j] = (m[j][i] + m[i][j]) * t; q[k] = (m[k][i] + m[i][k]) * t;
  }
}

std::string dir_of(const std::string& path) { size_t s = path.find_last_of('/'); return s == std::string::npos ? std::string() : path.substr(0, s + 1); }

struct Frame { double stamp; dvo::core::RgbdImagePyramidPtr pyramid; dvo_b200_pyramid* rectified; };

// --distortion: the frames go through a rectifier (dvo_b200_rectifier) on a context of this program's own, and the pairs
// are aligned through the C ABI with the tracker's configuration, as DenseTracker::matchBatch aligns them.
struct Rectified {
  dvo_b200_ctx* ctx = nullptr;
  dvo_b200_rectifier* rect = nullptr;
  ~Rectified() {
    if (rect) dvo_b200_rectifier_release(rect);
    if (ctx) dvo_b200_destroy(ctx);
  }
};

}  // namespace

int main(int argc, char** argv) {
  std::string assoc, gt_path, out_path;
  float K[4] = {517.3f, 516.5f, 318.6f, 255.3f};     // TUM freiburg1 (benchmark_slam.cpp:384)
  int first = 3, last = 1, batch = 32, max_frames = -1;
  bool parse_only = false;
  bool distorted = false;
  double dist[5] = {0, 0, 0, 0, 0};   // k1 k2 p1 p2 k3 (plumb bob)
  for (int i = 1; i < argc; ++i) {
    const std::string a = argv[i];
    if (a == "--assoc" && i + 1 < argc) assoc = argv[++i];
    else if (a == "--groundtruth" && i + 1 < argc) gt_path = argv[++i];
    else if (a == "--out" && i + 1 < argc) out_path = argv[++i];
    else if (a == "--intrinsics" && i + 4 < argc) { for (int k = 0; k < 4; ++k) K[k] = float(std::atof(argv[++i])); }
    else if (a == "--first" && i + 1 < argc) first = std::atoi(argv[++i]);
    else if (a == "--last" && i + 1 < argc) last = std::atoi(argv[++i]);
    else if (a == "--batch" && i + 1 < argc) batch = std::max(1, std::atoi(argv[++i]));
    else if (a == "--max-frames" && i + 1 < argc) max_frames = std::atoi(argv[++i]);
    else if (a == "--parse-only") parse_only = true;
    else if (a == "--distortion" && i + 5 < argc) {
      distorted = true;
      for (int k = 0; k < 5; ++k) {
        char* end = nullptr;
        dist[k] = std::strtod(argv[++i], &end);
        if (end == argv[i] || *end) { std::fprintf(stderr, "tum_replay: --distortion takes five numbers k1 k2 p1 p2 k3\n"); return 2; }
      }
    }
    else { std::fprintf(stderr, "usage: tum_replay --assoc assoc.txt [--groundtruth gt.txt] [--out traj.txt] [--intrinsics fx fy ox oy]\n"
                                "                  [--distortion k1 k2 p1 p2 k3] [--first L] [--last L] [--batch N] [--max-frames N]\n"
                                "                  [--parse-only]\n"); return 2; }
  }
  if (assoc.empty()) { std::fprintf(stderr, "tum_replay: --assoc is required\n"); return 2; }
  std::vector<RgbdPair> pairs;
  if (!read_entries(assoc, pairs) || pairs.empty()) { std::fprintf(stderr, "tum_replay: no entries in %s\n", assoc.c_str()); return 2; }
  if (max_frames > 0 && int(pairs.size()) > max_frames) pairs.resize(max_frames);
  std::vector<Groundtruth> gt;
  if (!gt_path.empty() && !read_entries(gt_path, gt)) { std::fprintf(stderr, "tum_replay: cannot read %s\n", gt_path.c_str()); return 2; }
  const std::string folder = dir_of(assoc);

  // first pose: closest ground-truth entry at or after the first RGB stamp (findClosestEntry, tools.h:68-82)
  dvo::core::AffineTransformd trajectory;
  trajectory.setIdentity();          // benchmark.cpp:399: identity unless ground truth provides the first pose
  size_t gt_first = 0;
  if (!gt.empty()) {
    while (gt_first + 1 < gt.size() && gt[gt_first].stamp < pairs.front().rgb_stamp) ++gt_first;
    trajectory = pose_from(gt[gt_first]);
  }

  std::string why;
  if (parse_only) {
    Image rgb, depth;
    if (!load_png(folder + pairs[0].rgb_file, rgb, why) || !load_png(folder + pairs[0].depth_file, depth, why)) { std::fprintf(stderr, "tum_replay: %s\n", why.c_str()); return 2; }
    cv::Mat grey, z;
    if (!to_grey_f32(rgb, grey, why) || !to_depth_f32(depth, 1.0f / 5000.0f, z, why)) { std::fprintf(stderr, "tum_replay: %s\n", why.c_str()); return 2; }
    double gsum = 0, zsum = 0; long long znan = 0;
    for (size_t i = 0; i < grey.total(); ++i) gsum += grey.ptr<float>()[i];
    for (size_t i = 0; i < z.total(); ++i) { float v = z.ptr<float>()[i]; if (v != v) ++znan; else zsum += v; }
    double q[4];
    quaternion_of(trajectory, q);
    std::printf("{\"pairs\": %zu, \"groundtruth\": %zu, \"gt_first\": %zu, \"first_stamp\": \"%s\", \"rgb\": [%d, %d, %d, %d], \"depth\": [%d, %d, %d, %d], "
                "\"grey_sum\": %.17g, \"depth_sum\": %.17g, \"depth_nan\": %lld, \"pose0\": [%.17g, %.17g, %.17g, %.17g, %.17g, %.17g, %.17g]%s}\n",
                pairs.size(), gt.size(), gt_first, stamp_text(pairs[0].rgb_stamp).c_str(), rgb.w, rgb.h, rgb.channels, rgb.bits, depth.w, depth.h,
                depth.channels, depth.bits, gsum, zsum, znan, trajectory.matrix()(0, 3), trajectory.matrix()(1, 3), trajectory.matrix()(2, 3), q[0], q[1], q[2], q[3],
                distorted ? (", \"distortion\": [" + std::to_string(dist[0]) + ", " + std::to_string(dist[1]) + ", " + std::to_string(dist[2]) + ", " +
                             std::to_string(dist[3]) + ", " + std::to_string(dist[4]) + "]").c_str() : "");
    return 0;
  }

  std::ofstream traj_file;
  if (!out_path.empty()) { traj_file.open(out_path.c_str()); if (!traj_file) { std::fprintf(stderr, "tum_replay: cannot write %s\n", out_path.c_str()); return 2; } }
  std::ostream& traj_out = out_path.empty() ? std::cout : traj_file;
  traj_out.precision(17);

  dvo::DenseTracker::Config cfg = dvo::DenseTracker::getDefaultConfig();
  cfg.FirstLevel = first; cfg.LastLevel = last;
  std::vector<Frame> frames;     // frames[0] is the reference of the first pending alignment
  size_t aligned = 0, failed = 0;
  double match_ms = 0.0;
  try {
    Image first_rgb;
    if (!load_png(folder + pairs[0].rgb_file, first_rgb, why)) { std::fprintf(stderr, "tum_replay: %s\n", why.c_str()); return 2; }
    dvo::core::RgbdCameraPyramid camera(size_t(first_rgb.w), size_t(first_rgb.h), dvo::core::IntrinsicMatrix::create(K[0], K[1], K[2], K[3]));
    dvo::DenseTracker tracker(cfg);
    Rectified rectified;
    dvo_b200_config ccfg;
    if (distorted) {   // one rectifier for the sequence: K_new = --intrinsics, the frames' size
      const int w = first_rgb.w, h = first_rgb.h;
      const double Kd[4] = {K[0], K[1], K[2], K[3]};
      std::vector<float> mx(size_t(w) * h), my(size_t(w) * h);
      const char* dev = std::getenv("DVO_B200_DEVICE");
      if (dvo_b200_undistort_map(w, h, Kd, dist, Kd, mx.data(), my.data()) != 0 ||
          dvo_b200_create(dev ? std::atoi(dev) : 0, 0, &rectified.ctx) != 0 ||
          dvo_b200_rectifier_create(rectified.ctx, w, h, w, h, mx.data(), my.data(), K, &rectified.rect) != 0) {
        std::fprintf(stderr, "tum_replay: cannot set up the rectifier: %s\n", rectified.ctx ? dvo_b200_last_error(rectified.ctx) : "no CUDA device");
        return 3;
      }
      dvo_b200_config_default(&ccfg);   // the fields DenseTracker::matchBatch passes
      ccfg.first_level = cfg.FirstLevel; ccfg.last_level = cfg.LastLevel; ccfg.max_iterations_per_level = cfg.MaxIterationsPerLevel;
      ccfg.use_initial_estimate = 0; ccfg.precision = cfg.Precision; ccfg.mu = cfg.Mu;
      ccfg.intensity_derivative_threshold = cfg.IntensityDerivativeThreshold; ccfg.depth_derivative_threshold = cfg.DepthDerivativeThreshold;
    }
    for (size_t next = 0; next < pairs.size();) {
      // load up to `batch` new frames behind the current reference
      while (next < pairs.size() && frames.size() < size_t(batch) + 1) {
        Image rgb, depth;
        cv::Mat grey, z;
        if (!load_png(folder + pairs[next].rgb_file, rgb, why) || !load_png(folder + pairs[next].depth_file, depth, why) ||
            !to_grey_f32(rgb, grey, why) || !to_depth_f32(depth, 1.0f / 5000.0f, z, why)) {
          std::fprintf(stderr, "tum_replay: skipping frame %zu: %s\n", next, why.c_str());   // load() returns a null pointer -> `continue`
          ++next;
          continue;
        }
        Frame f = {pairs[next].rgb_stamp, dvo::core::RgbdImagePyramidPtr(), nullptr};
        if (distorted) {
          if (grey.cols != first_rgb.w || grey.rows != first_rgb.h) { std::fprintf(stderr, "tum_replay: frame %zu: size differs from the first frame\n", next); return 2; }
          if (dvo_b200_pyramid_create_rectified_batch(rectified.ctx, rectified.rect, 1, DVO_B200_INPUT_FLOAT32, grey.ptr<float>(), z.ptr<float>(), 0.f,
                                                      nullptr, DVO_B200_MASK_ROLE_REFERENCE, grey.cols, grey.rows, int(cfg.getNumLevels()),
                                                      &f.rectified) != 0 ||
              dvo_b200_synchronize(rectified.ctx) != 0) {   // the frame's host images go out of scope
            std::fprintf(stderr, "tum_replay: %s\n", dvo_b200_last_error(rectified.ctx));
            return 3;
          }
        } else {
          f.pyramid = camera.create(grey, z);
        }
        frames.push_back(f);
        ++next;
      }
      if (frames.size() < 2) break;
      std::vector<dvo::DenseTracker::Result> results(frames.size() - 1);
      const auto t0 = std::chrono::steady_clock::now();
      if (distorted) {
        std::vector<dvo_b200_pyramid*> references, currents;
        for (size_t i = 1; i < frames.size(); ++i) { references.push_back(frames[i - 1].rectified); currents.push_back(frames[i].rectified); }
        std::vector<dvo_b200_result> raw(references.size());
        if (dvo_b200_match_batch(rectified.ctx, &ccfg, int(raw.size()), references.data(), currents.data(), nullptr, raw.data(), nullptr, 0) != 0) {
          std::fprintf(stderr, "tum_replay: dvo_b200_match_batch: %s\n", dvo_b200_last_error(rectified.ctx));
          return 3;
        }
        for (size_t i = 0; i < raw.size(); ++i) {   // what Result::isNaN and the trajectory read, as fill_result copies them
          for (int a = 0; a < 4; ++a)
            for (int b = 0; b < 4; ++b) results[i].Transformation.matrix()(a, b) = raw[i].transformation[a * 4 + b];
          for (int a = 0; a < 6; ++a)
            for (int b = 0; b < 6; ++b) results[i].Information(a, b) = raw[i].information[a * 6 + b];
        }
        for (size_t i = 0; i + 1 < frames.size(); ++i) dvo_b200_pyramid_release(frames[i].rectified);   // the last one is the next reference
      } else {
        std::vector<dvo::core::RgbdImagePyramid*> references, currents;
        for (size_t i = 1; i < frames.size(); ++i) { references.push_back(frames[i - 1].pyramid.get()); currents.push_back(frames[i].pyramid.get()); }
        tracker.matchBatch(references, currents, results);
      }
      match_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
      for (size_t i = 0; i < results.size(); ++i) {
        if (results[i].isNaN()) { ++failed; results[i].setIdentity(); }
        trajectory = trajectory * results[i].Transformation;            // benchmark.cpp:463
        double q[4];
        quaternion_of(trajectory, q);
        traj_out << stamp_text(frames[i + 1].stamp) << " " << trajectory.matrix()(0, 3) << " " << trajectory.matrix()(1, 3) << " " << trajectory.matrix()(2, 3)
                 << " " << q[0] << " " << q[1] << " " << q[2] << " " << q[3] << " " << std::endl;
        ++aligned;
      }
      Frame keep = frames.back();
      frames.clear();
      frames.push_back(keep);
    }
    if (distorted && !frames.empty()) dvo_b200_pyramid_release(frames.back().rectified);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  double q[4];
  quaternion_of(trajectory, q);
  std::fprintf(stderr, "{\"frames\": %zu, \"alignments\": %zu, \"failed\": %zu, \"match_ms\": %.3f, \"alignments_per_s\": %.1f, "
                       "\"final_pose\": [%.9g, %.9g, %.9g, %.9g, %.9g, %.9g, %.9g]}\n",
               pairs.size(), aligned, failed, match_ms, match_ms > 0 ? 1e3 * double(aligned) / match_ms : 0.0, trajectory.matrix()(0, 3),
               trajectory.matrix()(1, 3), trajectory.matrix()(2, 3), q[0], q[1], q[2], q[3]);
  return 0;
}
