// DenseTracker::matchWithWeights through the C++ adapter, for tests/test_gpu_weight_maps.py: reads a raw float32 pair (I_ref,
// Z_ref, I_cur, Z_cur, h x w each), aligns it with match() and with matchWithWeights() on levels 3..1, writes the weight map
// (rows x cols float32) to out.bin and prints the pose, whether both Results are equal, and the map's size as JSON.  With
// priors.bin (two row-major 6 x 6 float64 priors) it also aligns the pair with matchWithPrior() under the first prior and, as a
// batch of two pairs, with the matchBatch() overload under both, and prints those poses as "prior_T" and "batch_T".
// Exit 3 = no CUDA device.
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
  if (argc < 9) { std::fprintf(stderr, "usage: weights_adapter pair.bin w h fx fy ox oy out.bin [priors.bin]\n"); return 2; }
  const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
  dvo::core::IntrinsicMatrix K = dvo::core::IntrinsicMatrix::create(float(std::atof(argv[4])), float(std::atof(argv[5])),
                                                                     float(std::atof(argv[6])), float(std::atof(argv[7])));
  std::ifstream f(argv[1], std::ios::binary);
  if (!f) { std::fprintf(stderr, "cannot open %s\n", argv[1]); return 2; }
  cv::Mat Ir = load_plane(f, w, h), Zr = load_plane(f, w, h), Ic = load_plane(f, w, h), Zc = load_plane(f, w, h);
  std::vector<dvo::core::Matrix6d> priors;
  if (argc >= 10) {
    std::ifstream fp(argv[9], std::ios::binary);
    if (!fp) { std::fprintf(stderr, "cannot open %s\n", argv[9]); return 2; }
    priors.resize(2);
    for (int j = 0; j < 2; ++j) {
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
  dvo::DenseTracker::Result plain, with_weights, with_prior;
  std::vector<dvo::DenseTracker::Result> batch;
  cv::Mat weights;
  bool ok = false, ok_prior = false, ok_batch = false;
  try {
    tracker.match(*reference, *current, plain);
    ok = tracker.matchWithWeights(*reference, *current, with_weights, weights);
    if (!priors.empty()) {
      ok_prior = tracker.matchWithPrior(*reference, *current, priors[0], with_prior);
      std::vector<dvo::core::RgbdImagePyramid*> refs(2, reference.get()), curs(2, current.get());
      ok_batch = tracker.matchBatch(refs, curs, priors, batch);
    }
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
  if (!priors.empty()) {
    std::printf("], \"prior_ok\": %d, \"batch_ok\": %d, \"prior_T\": [", int(ok_prior), int(ok_batch));
    for (int i = 0; i < 4; ++i)
      for (int j = 0; j < 4; ++j) std::printf("%s%.17g", (i + j) ? ", " : "", with_prior.Transformation.matrix()(i, j));
    std::printf("], \"batch_T\": [");
    for (size_t p = 0; p < batch.size(); ++p)
      for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) std::printf("%s%.17g", (p + i + j) ? ", " : "", batch[p].Transformation.matrix()(i, j));
  }
  std::printf("]}\n");
  return 0;
}
