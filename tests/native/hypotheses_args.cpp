// The checks and the selection rule of csrc/hypotheses_args.h on the host, for tests/test_hypotheses_host.py: a shared library
// with C entry points.
#include <cstring>

#include "hypotheses_args.h"

extern "C" {

// has_cfg = 0: a NULL cfg; has_results / has_best = 0: a NULL results / best.  Writes the refusal (or "") to msg.
int hyp_check(int has_cfg, int first_level, int last_level, int use_initial_estimate, int n, int k, const double* hypotheses,
              int screen_level, double min_constraint_ratio, int has_results, int has_best, char* msg, int cap) {
  dvo_b200_config cfg{};
  cfg.first_level = first_level; cfg.last_level = last_level; cfg.use_initial_estimate = use_initial_estimate;
  dvo_b200_result result{};
  int32_t best = 0;
  const std::string why = dvo_b200::hypotheses_args_error(has_cfg ? &cfg : nullptr, n, k, hypotheses, screen_level, min_constraint_ratio,
                                                          has_results ? &result : nullptr, has_best ? &best : nullptr);
  std::strncpy(msg, why.c_str(), (size_t)cap - 1);
  msg[cap - 1] = 0;
  return why.empty() ? 0 : 1;
}

double hyp_score(int has_increment, long long inc_constraints, long long valid_pixels, double inc_log_likelihood, double min_ratio) {
  return dvo_b200::hypothesis_score(has_increment, inc_constraints, valid_pixels, inc_log_likelihood, min_ratio);
}

int hyp_pick(const double* scores, int k) { return dvo_b200::pick_hypothesis(scores, k); }

}  // extern "C"
