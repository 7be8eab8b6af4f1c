// The checks and the shard slicing of dvo_b200_match_batch_modes_device / _modes_sharded (csrc/modes_args.h) on the host, for
// tests/test_modes_multi_gpu_host.py: a shared library with two C entry points.
#include <cstring>
#include <vector>

#include "modes_args.h"

namespace {

// fake addresses: pointer i of a call lies at kBase * (i + 1)
constexpr uintptr_t kBase = 0x100000000ull;
template <typename T>
T* fake(int i) { return reinterpret_cast<T*>(kBase * (uintptr_t)(i + 1)); }

}  // namespace

extern "C" {

// The slice [b, e) of a batch of n pairs with k hypotheses, max_log log entries per pair and maps whose weight plane has
// weight_image_bytes and mask plane mask_image_bytes per pair.  off[] receives the byte offset of each sliced pointer from
// the unsliced one, in the order refs, curs, hypotheses, prior, photometric_init, photometric, screen_photometric, results,
// best, scores, screen_results, iteration_stats, weight, mask, estimate, precision; returns the slice's n.
int ms_slice(int n, int k, int max_log, long long b, long long e, long long weight_image_bytes, long long mask_image_bytes, long long* off) {
  dvo_b200::ModesArgs a;
  a.n = n; a.k = k; a.max_log = max_log;
  a.refs = fake<dvo_b200_pyramid* const>(0); a.curs = fake<dvo_b200_pyramid* const>(1);
  a.hypotheses = fake<const double>(2); a.prior = fake<const double>(3); a.ab_init = fake<const double>(4);
  a.ab = fake<double>(5); a.screen_ab = fake<double>(6); a.results = fake<dvo_b200_result>(7); a.best = fake<int32_t>(8);
  a.scores = fake<double>(9); a.screen_results = fake<dvo_b200_result>(10); a.iter_stats = fake<dvo_b200_iteration_stats>(11);
  dvo_b200_weight_maps m{};
  m.weight = {fake<void>(12), 64, weight_image_bytes};
  m.mask = {fake<void>(13), 32, mask_image_bytes};
  m.estimate = fake<double>(14); m.precision = fake<float>(15);
  a.maps = &m;
  dvo_b200_weight_maps sm;
  const dvo_b200::ModesArgs s = dvo_b200::shard_slice(a, b, e, &sm);
  const void* before[16] = {a.refs, a.curs, a.hypotheses, a.prior, a.ab_init, a.ab, a.screen_ab, a.results, a.best, a.scores,
                            a.screen_results, a.iter_stats, m.weight.data, m.mask.data, m.estimate, m.precision};
  const void* after[16] = {s.refs, s.curs, s.hypotheses, s.prior, s.ab_init, s.ab, s.screen_ab, s.results, s.best, s.scores,
                           s.screen_results, s.iter_stats, s.maps->weight.data, s.maps->mask.data, s.maps->estimate, s.maps->precision};
  for (int i = 0; i < 16; ++i) off[i] = (long long)((const char*)after[i] - (const char*)before[i]);
  return s.n;
}

// Every up-front check of the form (0: device, 1: sharded) over ndev devices.  Pyramids: ref i is views[i], cur i is
// views[n + i], each {levels, device, w0, h0}, level l of size (w0 >> l) x (h0 >> l).  Outputs: an address per output of
// modes_outputs' order (photometric, screen_photometric, results, best, scores, screen_results, iteration_stats), 0 = NULL.
// The fake's memory: [dev_begin, dev_end) is device memory of device 0, everything else host memory.  Writes the refusal (or
// "") to msg and returns the status it carries (0 if accepted).
int ms_check(int form, int ndev, const int* devices, int first_level, int last_level, double mu, int use_initial_estimate, int n,
             const int* views, int k, const double* hypotheses, int screen_level, const double* prior, const double* ab_init,
             const long long* outputs, int max_log, const dvo_b200_weight_maps* maps, long long dev_begin, long long dev_end, char* msg,
             int cap) {
  dvo_b200_config cfg{};
  cfg.first_level = first_level; cfg.last_level = last_level; cfg.max_iterations_per_level = 20; cfg.mu = mu;
  cfg.use_initial_estimate = use_initial_estimate;
  std::vector<dvo_b200_pyramid*> pyr(2 * (size_t)(n > 0 ? n : 0));
  for (size_t i = 0; i < pyr.size(); ++i) pyr[i] = fake<dvo_b200_pyramid>((int)i + 100);
  auto view = [&](const dvo_b200_pyramid* p, int level) {
    const int* v = views + 4 * ((uintptr_t)p / kBase - 101);
    const bool has = level >= 0 && level < v[0];
    return dvo_b200::PyramidView{v[0], v[1], v[2], v[3], has ? v[2] >> level : 0, has ? v[3] >> level : 0};
  };
  auto where = [&](const void* p) {
    const long long a = (long long)(uintptr_t)p;
    return a >= dev_begin && a < dev_end ? dvo_b200::PtrWhere{dvo_b200::kPtrDevice, 0} : dvo_b200::PtrWhere{dvo_b200::kPtrHost, -1};
  };
  dvo_b200::ModesArgs a;
  a.cfg = &cfg; a.n = n; a.refs = pyr.data(); a.curs = pyr.data() + (n > 0 ? n : 0); a.k = k; a.hypotheses = hypotheses;
  a.screen_level = screen_level; a.prior = prior; a.ab_init = ab_init;
  a.ab = (double*)(uintptr_t)outputs[0]; a.screen_ab = (double*)(uintptr_t)outputs[1]; a.results = (dvo_b200_result*)(uintptr_t)outputs[2];
  a.best = (int32_t*)(uintptr_t)outputs[3]; a.scores = (double*)(uintptr_t)outputs[4];
  a.screen_results = (dvo_b200_result*)(uintptr_t)outputs[5]; a.iter_stats = (dvo_b200_iteration_stats*)(uintptr_t)outputs[6];
  a.max_log = max_log; a.maps = maps;
  int code = 0;
  const std::string why = dvo_b200::modes_args_error(a, form ? dvo_b200::kFormSharded : dvo_b200::kFormDevice, ndev, devices, view,
                                                     where, &code);
  std::strncpy(msg, why.c_str(), (size_t)cap - 1);
  msg[cap - 1] = 0;
  return why.empty() ? 0 : code;
}

}  // extern "C"
