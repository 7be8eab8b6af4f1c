// DenseTracker::matchWithHypotheses through the C++ adapter, for tests/test_gpu_hypotheses.py: reads a raw float32 pair (I_ref,
// Z_ref, I_cur, Z_cur, h x w each) and k row-major 4 x 4 hypotheses (k * 16 float64), aligns on levels 3..1 with screen level 2,
// tries once more with screen level 0 (outside [LastLevel, FirstLevel]: refused) and prints both outcomes, the chosen index
// and the pose as JSON.  With priors.bin (k row-major 6 x 6 float64 priors, one per start) and out.bin it also aligns through the
// overload with priors and a weight map, writes the map (rows x cols float32) to out.bin and prints that outcome, chosen index
// and pose as "prior_ok", "prior_best" and "prior_T".  Exit 3 = no CUDA device.
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
  if (argc < 10) { std::fprintf(stderr, "usage: hypotheses_adapter pair.bin w h fx fy ox oy hypotheses.bin k [priors.bin out.bin]\n"); return 2; }
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
  std::vector<dvo::core::Matrix6d> priors;
  if (argc >= 12) {
    std::ifstream fp(argv[10], std::ios::binary);
    if (!fp) { std::fprintf(stderr, "cannot open %s\n", argv[10]); return 2; }
    priors.resize((size_t)k);
    for (int j = 0; j < k; ++j) {
      double L[36];
      fp.read(reinterpret_cast<char*>(L), sizeof(L));
      for (int a = 0; a < 6; ++a)
        for (int b = 0; b < 6; ++b) priors[(size_t)j](a, b) = L[a * 6 + b];
    }
  }
  dvo::core::RgbdCameraPyramid camera(w, h, K);
  dvo::core::RgbdImagePyramidPtr reference = camera.create(Ir, Zr), current = camera.create(Ic, Zc);
  dvo::DenseTracker::Config cfg = dvo::DenseTracker::getDefaultConfig();
  cfg.FirstLevel = 3;
  cfg.LastLevel = 1;
  cfg.MaxIterationsPerLevel = 50;
  cfg.Precision = 1e-4;
  dvo::DenseTracker tracker(cfg);
  dvo::DenseTracker::Result result, refused, with_prior;
  int best = -1, best_refused = -1, best_prior = -1;
  bool ok = false, ok_refused = true, ok_prior = false;
  cv::Mat weights;
  try {
    ok = tracker.matchWithHypotheses(*reference, *current, initial, 2, result, &best);
    ok_refused = tracker.matchWithHypotheses(*reference, *current, initial, 0, refused, &best_refused);
    if (!priors.empty()) ok_prior = tracker.matchWithHypotheses(*reference, *current, initial, priors, 2, with_prior, &best_prior, 0.0, &weights);
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  std::printf("{\"ok\": %d, \"refused_ok\": %d, \"refused_best\": %d, \"best\": %d, \"levels\": %d, \"T\": [", int(ok), int(ok_refused),
              best_refused, best, int(result.Statistics.Levels.size()));
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) std::printf("%s%.17g", (i + j) ? ", " : "", result.Transformation.matrix()(i, j));
  if (!priors.empty()) {
    std::ofstream o(argv[11], std::ios::binary);
    o.write(reinterpret_cast<const char*>(weights.ptr<float>()), sizeof(float) * size_t(weights.rows) * weights.cols);
    std::printf("], \"prior_ok\": %d, \"prior_best\": %d, \"rows\": %d, \"cols\": %d, \"prior_T\": [", int(ok_prior), best_prior,
                weights.rows, weights.cols);
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) std::printf("%s%.17g", (i + j) ? ", " : "", with_prior.Transformation.matrix()(i, j));
  }
  std::printf("]}\n");
  return 0;
}
