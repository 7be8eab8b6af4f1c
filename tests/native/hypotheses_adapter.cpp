// DenseTracker::matchWithHypotheses through the C++ adapter, for tests/test_gpu_hypotheses.py: reads a raw float32 pair (I_ref,
// Z_ref, I_cur, Z_cur, h x w each) and k row-major 4 x 4 hypotheses (k * 16 float64), aligns on levels 3..1 with screen level 2,
// tries once more with screen level 0 (outside [LastLevel, FirstLevel]: refused) and prints both outcomes, the chosen index
// and the pose as JSON.  Exit 3 = no CUDA device.
#include <cstdio>
#include <cstdlib>
#include <exception>
#include <fstream>
#include <vector>

#include "dvo/dense_tracking.h"

static cv::Mat load_plane(std::ifstream& f, int w, int h) {
  cv::Mat m(h, w, CV_32FC1);
  f.read(reinterpret_cast<char*>(m.ptr<float>()), sizeof(float) * size_t(w) * h);
  return m;
}

int main(int argc, char** argv) {
  if (argc < 10) { std::fprintf(stderr, "usage: hypotheses_adapter pair.bin w h fx fy ox oy hypotheses.bin k\n"); return 2; }
  const int w = std::atoi(argv[2]), h = std::atoi(argv[3]), k = std::atoi(argv[9]);
  dvo::core::IntrinsicMatrix K = dvo::core::IntrinsicMatrix::create(float(std::atof(argv[4])), float(std::atof(argv[5])),
                                                                     float(std::atof(argv[6])), float(std::atof(argv[7])));
  std::ifstream f(argv[1], std::ios::binary);
  std::ifstream fh(argv[8], std::ios::binary);
  if (!f || !fh) { std::fprintf(stderr, "cannot open the inputs\n"); return 2; }
  cv::Mat Ir = load_plane(f, w, h), Zr = load_plane(f, w, h), Ic = load_plane(f, w, h), Zc = load_plane(f, w, h);
  std::vector<dvo::core::AffineTransformd> initial((size_t)k);
  for (int j = 0; j < k; ++j) {
    double T[16];
    fh.read(reinterpret_cast<char*>(T), sizeof(T));
    for (int a = 0; a < 4; ++a)
      for (int b = 0; b < 4; ++b) initial[(size_t)j].matrix()(a, b) = T[a * 4 + b];
  }
  dvo::core::RgbdCameraPyramid camera(w, h, K);
  dvo::core::RgbdImagePyramidPtr reference = camera.create(Ir, Zr), current = camera.create(Ic, Zc);
  dvo::DenseTracker::Config cfg = dvo::DenseTracker::getDefaultConfig();
  cfg.FirstLevel = 3;
  cfg.LastLevel = 1;
  cfg.MaxIterationsPerLevel = 50;
  cfg.Precision = 1e-4;
  dvo::DenseTracker tracker(cfg);
  dvo::DenseTracker::Result result, refused;
  int best = -1, best_refused = -1;
  bool ok = false, ok_refused = true;
  try {
    ok = tracker.matchWithHypotheses(*reference, *current, initial, 2, result, &best);
    ok_refused = tracker.matchWithHypotheses(*reference, *current, initial, 0, refused, &best_refused);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  std::printf("{\"ok\": %d, \"refused_ok\": %d, \"refused_best\": %d, \"best\": %d, \"levels\": %d, \"T\": [", int(ok), int(ok_refused),
              best_refused, best, int(result.Statistics.Levels.size()));
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) std::printf("%s%.17g", (i + j) ? ", " : "", result.Transformation.matrix()(i, j));
  std::printf("]}\n");
  return 0;
}
