// The checks of csrc/prior_args.h on the host, for tests/test_prior_host.py: a shared library with one C entry point.
#include <cstring>

#include "prior_args.h"

extern "C" {

// has_cfg = 0: a NULL cfg; has_ab_init / has_ab: photometric_init / photometric non-NULL.  Writes the refusal (or "") to msg.
int prior_check(int has_cfg, double mu, int n, const double* prior, int has_ab_init, int has_ab, char* msg, int cap) {
  dvo_b200_config cfg{};
  cfg.mu = mu;
  double ab[2] = {1.0, 0.0};
  const std::string why = dvo_b200::prior_args_error(has_cfg ? &cfg : nullptr, n, prior, has_ab_init ? ab : nullptr,
                                                     has_ab ? ab : nullptr);
  std::strncpy(msg, why.c_str(), (size_t)cap - 1);
  msg[cap - 1] = 0;
  return why.empty() ? 0 : 1;
}

}  // extern "C"
