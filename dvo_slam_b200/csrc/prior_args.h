// prior_args.h -- the checks of a motion prior (dvo_b200_match_batch_prior) that need no CUDA call.  Plain C++ without CUDA,
// so that they can be built and run on the host alone (tests/native/prior_args.cpp).  capi.cu runs them before anything is
// staged, uploaded or launched.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <string>

#include "../../include/dvo_b200.h"

namespace dvo_b200 {

// The eigenvalues of a symmetric 6 x 6 (row-major) by cyclic Jacobi rotations in fp64, unordered.
inline void eigenvalues6(const double S[36], double ev[6]) {
  double a[36];
  for (int i = 0; i < 36; ++i) a[i] = S[i];
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = 0; i < 6; ++i) {
      diag += a[i * 6 + i] * a[i * 6 + i];
      for (int j = i + 1; j < 6; ++j) off += a[i * 6 + j] * a[i * 6 + j];
    }
    if (off <= 1e-30 * diag || off == 0.0) break;
    for (int p = 0; p < 5; ++p)
      for (int q = p + 1; q < 6; ++q) {
        const double apq = a[p * 6 + q];
        if (apq == 0.0) continue;
        const double theta = (a[q * 6 + q] - a[p * 6 + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 6; ++k) {   // A <- A J, then A <- J^T A
          const double akp = a[k * 6 + p], akq = a[k * 6 + q];
          a[k * 6 + p] = c * akp - s * akq;
          a[k * 6 + q] = s * akp + c * akq;
        }
        for (int k = 0; k < 6; ++k) {
          const double apk = a[p * 6 + k], aqk = a[q * 6 + k];
          a[p * 6 + k] = c * apk - s * aqk;
          a[q * 6 + k] = s * apk + c * aqk;
        }
      }
  }
  for (int i = 0; i < 6; ++i) ev[i] = a[i * 6 + i];
}

// Why the prior of one pair is refused, or "" if it is accepted: every entry finite, exactly symmetric, and no eigenvalue
// below -1e-9 max(1, max |Lambda_ij|).  Positive semi-definite and rank-deficient priors are accepted.
inline std::string prior_matrix_error(const double L[36]) {
  double amax = 0.0;
  for (int i = 0; i < 36; ++i) {
    if (!std::isfinite(L[i])) return "is not finite";
    amax = std::fmax(amax, std::fabs(L[i]));
  }
  for (int i = 0; i < 6; ++i)
    for (int j = i + 1; j < 6; ++j)
      if (L[i * 6 + j] != L[j * 6 + i]) return "is not symmetric";
  double ev[6];
  eigenvalues6(L, ev);
  const double tol = -1e-9 * std::fmax(1.0, amax);
  for (int i = 0; i < 6; ++i)
    if (!(ev[i] >= tol)) return "is not positive semi-definite";
  return "";
}

// The checks of dvo_b200_match_batch_prior beyond those of dvo_b200_match_batch[_photometric], in this order: a NULL
// prior_information, photometric_init without photometric, cfg->mu != 0, then each pair's matrix.  A NULL cfg or n <= 0 is
// left to the batch checks that follow.  Returns "" or the message, prefixed with "match_batch_prior: ".
inline std::string prior_args_error(const dvo_b200_config* cfg, int32_t n, const double* prior_information,
                                    const double* photometric_init, const double* photometric) {
  const std::string fn = "match_batch_prior: ";
  if (!prior_information) return fn + "prior_information is null";
  if (photometric_init && !photometric) return fn + "photometric_init without photometric";
  if (cfg && cfg->mu != 0.0) return fn + "cfg->mu must be 0: the prior replaces mu I";
  if (!cfg) return "";
  for (int32_t p = 0; p < n; ++p) {
    const std::string why = prior_matrix_error(prior_information + (size_t)p * 36);
    if (!why.empty()) return fn + "prior_information of pair " + std::to_string(p) + " " + why;
  }
  return "";
}

}  // namespace dvo_b200
