// DenseTracker::matchWithWeights through the C++ adapter, for tests/test_gpu_weight_maps.py: reads a raw float32 pair (I_ref,
// Z_ref, I_cur, Z_cur, h x w each), aligns it with match() and with matchWithWeights() on levels 3..1, writes the weight map
// (rows x cols float32) to out.bin and prints the pose, whether both Results are equal, and the map's size as JSON.
// Exit 3 = no CUDA device.
#include <cstdio>
#include <cstdlib>
#include <exception>
#include <fstream>

#include "dvo/dense_tracking.h"

static cv::Mat load_plane(std::ifstream& f, int w, int h) {
  cv::Mat m(h, w, CV_32FC1);
  f.read(reinterpret_cast<char*>(m.ptr<float>()), sizeof(float) * size_t(w) * h);
  return m;
}

int main(int argc, char** argv) {
  if (argc < 9) { std::fprintf(stderr, "usage: weights_adapter pair.bin w h fx fy ox oy out.bin\n"); return 2; }
  const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
  dvo::core::IntrinsicMatrix K = dvo::core::IntrinsicMatrix::create(float(std::atof(argv[4])), float(std::atof(argv[5])),
                                                                     float(std::atof(argv[6])), float(std::atof(argv[7])));
  std::ifstream f(argv[1], std::ios::binary);
  if (!f) { std::fprintf(stderr, "cannot open %s\n", argv[1]); return 2; }
  cv::Mat Ir = load_plane(f, w, h), Zr = load_plane(f, w, h), Ic = load_plane(f, w, h), Zc = load_plane(f, w, h);
  dvo::core::RgbdCameraPyramid camera(w, h, K);
  dvo::core::RgbdImagePyramidPtr reference = camera.create(Ir, Zr), current = camera.create(Ic, Zc);
  dvo::DenseTracker::Config cfg = dvo::DenseTracker::getDefaultConfig();
  cfg.FirstLevel = 3;
  cfg.LastLevel = 1;
  cfg.MaxIterationsPerLevel = 50;
  cfg.Precision = 1e-4;
  dvo::DenseTracker tracker(cfg);
  dvo::DenseTracker::Result plain, with_weights;
  cv::Mat weights;
  bool ok = false;
  try {
    tracker.match(*reference, *current, plain);
    ok = tracker.matchWithWeights(*reference, *current, with_weights, weights);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  bool same = plain.LogLikelihood == with_weights.LogLikelihood;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) same = same && plain.Transformation.matrix()(i, j) == with_weights.Transformation.matrix()(i, j);
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j < 6; ++j) same = same && plain.Information(i, j) == with_weights.Information(i, j);
  std::ofstream o(argv[8], std::ios::binary);
  o.write(reinterpret_cast<const char*>(weights.ptr<float>()), sizeof(float) * size_t(weights.rows) * weights.cols);
  std::printf("{\"ok\": %d, \"same\": %d, \"rows\": %d, \"cols\": %d, \"T\": [", int(ok), int(same), weights.rows, weights.cols);
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) std::printf("%s%.17g", (i + j) ? ", " : "", with_weights.Transformation.matrix()(i, j));
  std::printf("]}\n");
  return 0;
}
