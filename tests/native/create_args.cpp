// The argument checks of csrc/create_args.h on the host, for tests/test_create_args_host.py.
//
// One case per input line:
//   fn remap device ctx out image depth n format roles width height levels
//      rect rect_in_w rect_in_h rect_w rect_h rect_fx reg reg_w reg_h reg_fx
// ctx / out / image / depth: 1 for a pointer, 0 for NULL.  rect / reg: 0 none, 1 of the calling context, 2 of another
// context; their K is (fx, 500, 320, 240).  One line per case: "ok", or the refusal.
#include <iostream>
#include <sstream>
#include <string>

#include "create_args.h"

using namespace dvo_b200;

int main() {
  char own_byte = 0, other_byte = 0, frame = 0;
  dvo_b200_ctx* own = reinterpret_cast<dvo_b200_ctx*>(&own_byte);
  dvo_b200_ctx* other = reinterpret_cast<dvo_b200_ctx*>(&other_byte);
  dvo_b200_device_plane plane{&frame, 1, 1};
  dvo_b200_pyramid* handles[1] = {nullptr};
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string fn;
    int ctx, out, image, depth, rect, reg, rect_fx, reg_fx;
    CreateArgs a;
    dvo_b200_rectifier r;
    dvo_b200_depth_registration g;
    if (!(in >> fn >> a.remap >> a.device >> ctx >> out >> image >> depth >> a.n >> a.format >> a.roles >> a.width >> a.height >>
          a.levels >> rect >> r.in_w >> r.in_h >> r.w >> r.h >> rect_fx >> reg >> g.w >> g.h >> reg_fx))
      return 1;
    a.fn = fn.c_str();
    r.ctx = rect == 1 ? own : other;
    g.ctx = reg == 1 ? own : other;
    const float K[4] = {500.f, 500.f, 320.f, 240.f};
    for (int i = 0; i < 4; ++i) { a.K[i] = K[i]; r.K[i] = K[i]; g.K[i] = K[i]; }
    r.K[0] = (float)rect_fx;
    g.K[0] = (float)reg_fx;
    g.dw = 320; g.dh = 240;
    a.rect = rect ? &r : nullptr;
    a.reg = reg ? &g : nullptr;
    if (a.device) {
      a.image_plane = image ? &plane : nullptr;
      a.depth_plane = depth ? &plane : nullptr;
    } else {
      a.image = image ? &frame : nullptr;
      a.depth = depth ? &frame : nullptr;
    }
    const std::string why = create_args_error(ctx ? own : nullptr, a, out ? handles : nullptr);
    std::cout << (why.empty() ? "ok" : why) << "\n";
  }
  return 0;
}
