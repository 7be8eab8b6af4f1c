// The checks of dvo_b200_match_batch_hypotheses_modes (csrc/hypotheses_args.h) on the host, for
// tests/test_hypotheses_modes_host.py: a shared library with one C entry point.
#include <cstring>

#include "hypotheses_args.h"

extern "C" {

// has_cfg = 0: a NULL cfg; has_photometric / has_screen_photometric: a non-NULL photometric / screen_photometric output;
// has_extent = 0: a batch the match would refuse (maps checked as for n = 0).  The fake's memory: [dev_begin, dev_end) is
// device memory of device 0, everything else host memory.  Writes the refusal (or "") to msg.
int hm_check(int has_cfg, int first_level, int last_level, double mu, int n, int k, const double* hypotheses, int screen_level,
             double min_constraint_ratio, const double* prior_information, const double* photometric_init, int has_photometric,
             int has_screen_photometric, const dvo_b200_weight_maps* maps, int has_extent, int w, int h, int w0, int h0,
             long long dev_begin, long long dev_end, char* msg, int cap) {
  dvo_b200_config cfg{};
  cfg.first_level = first_level; cfg.last_level = last_level; cfg.use_initial_estimate = 1; cfg.mu = mu;
  dvo_b200_result result{};
  int32_t best = 0;
  double photometric[2], screen_photometric[2];
  const dvo_b200::MapsExtent extent{w, h, w0, h0};
  auto where = [&](const void* p) {
    const long long a = (long long)(uintptr_t)p;
    return a >= dev_begin && a < dev_end ? dvo_b200::PtrWhere{dvo_b200::kPtrDevice, 0} : dvo_b200::PtrWhere{dvo_b200::kPtrHost, -1};
  };
  const std::string why = dvo_b200::hypotheses_modes_args_error(
      has_cfg ? &cfg : nullptr, n, k, hypotheses, screen_level, min_constraint_ratio, &result, &best, prior_information, photometric_init,
      has_photometric ? photometric : nullptr, has_screen_photometric ? screen_photometric : nullptr, maps, has_extent ? &extent : nullptr, 0,
      where);
  std::strncpy(msg, why.c_str(), (size_t)cap - 1);
  msg[cap - 1] = 0;
  return why.empty() ? 0 : 1;
}

}  // extern "C"
