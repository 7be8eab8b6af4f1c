// The checks of csrc/maps_args.h on the host, for tests/test_weight_maps_host.py: a shared library with one C entry point.
#include <cstring>

#include "maps_args.h"

extern "C" {

// The memory of the fake: regions[3 * i .. 3 * i + 2] = {first address, end address, kind * 16 + device}; every other
// address is host memory.  Writes the refusal (or "") to msg.
int maps_check(const dvo_b200_weight_maps* maps, int n, int w, int h, int w0, int h0, int device, const long long* regions,
               int nregions, char* msg, int cap) {
  auto where = [&](const void* p) {
    const long long a = (long long)(uintptr_t)p;
    for (int i = 0; i < nregions; ++i)
      if (a >= regions[3 * i] && a < regions[3 * i + 1])
        return dvo_b200::PtrWhere{int(regions[3 * i + 2] / 16), int(regions[3 * i + 2] % 16)};
    return dvo_b200::PtrWhere{dvo_b200::kPtrHost, -1};
  };
  const std::string why = dvo_b200::maps_args_error(maps, n, dvo_b200::MapsExtent{w, h, w0, h0}, device, where);
  std::strncpy(msg, why.c_str(), (size_t)cap - 1);
  msg[cap - 1] = 0;
  return why.empty() ? 0 : 1;
}

}  // extern "C"
