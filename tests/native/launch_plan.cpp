// The launch plan of csrc/launch_plan.h on the host, for tests/test_launch_plan_host.py.
//
// One case per input line:  grid npairs first last nlevels {h nbands nstrips} x nlevels [NAME=VALUE ...]
// where NAME=VALUE sets a DVO_B200_* plan override for this case only.  One JSON line per case:
// [[segment, ...] per launch], each segment an object with the fields of PlanSegment.
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "launch_plan.h"

using namespace dvo_b200;

int main() {
  const char* knobs[] = {"DVO_B200_NO_WALK", "DVO_B200_NO_FUSE", "DVO_B200_CONTIGUOUS", "DVO_B200_COARSE_TILES",
                         "DVO_B200_TAIL", "DVO_B200_STRIPS_PER_CTA", "DVO_B200_FINE_G"};
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    int grid, npairs, first, last, nlevels;
    if (!(in >> grid >> npairs >> first >> last >> nlevels) || nlevels > DVO_B200_MAX_LEVELS) return 1;
    LevelShape shape[DVO_B200_MAX_LEVELS];
    for (int l = 0; l < nlevels; ++l)
      if (!(in >> shape[l].h >> shape[l].nbands >> shape[l].nstrips)) return 1;
    for (const char* k : knobs) unsetenv(k);
    for (std::string kv; in >> kv;) {
      const size_t eq = kv.find('=');
      if (eq == std::string::npos) return 1;
      setenv(kv.substr(0, eq).c_str(), kv.substr(eq + 1).c_str(), 1);
    }
    const LaunchPlan p = make_launch_plan(shape, first, last, grid, npairs, plan_knobs_from_env());
    printf("[");
    for (int i = 0; i < p.nlaunch; ++i) {
      printf(i ? ", [" : "[");
      for (int s = 0; s < p.launch[i].nseg; ++s) {
        const PlanSegment& S = p.launch[i].seg[s];
        printf("%s{\"first_li\": %d, \"nlev\": %d, \"g\": %d, \"nsquads\": %d, \"strips_per_cta\": [", s ? ", " : "", S.first_li,
               S.nlev, S.g, S.nsquads);
        for (int k = 0; k < S.nlev; ++k) printf(k ? ", %d" : "%d", S.strips_per_cta[k]);
        printf("], \"pair_begin\": %d, \"npairs\": %d, \"hmax\": %d, \"cyclic\": %d}", S.pair_begin, S.npairs, S.hmax, S.cyclic);
      }
      printf("]");
    }
    printf("]\n");
  }
  return 0;
}
