// maps_args.h -- the checks of the output description of dvo_b200_match_batch_maps.  Plain C++ without CUDA, so that they can
// be built and run on the host alone (tests/native/maps_args.cpp): where a pointer lies is asked through `where`, which
// capi.cu answers with cudaPointerGetAttributes and the host test with a fake.  capi.cu runs them before anything is
// staged, uploaded or launched.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <string>

#include "../../include/dvo_b200.h"

namespace dvo_b200 {

// Where one byte lies, as cudaPointerGetAttributes reports it.
enum PtrKind { kPtrHost = 0, kPtrDevice = 1, kPtrManaged = 2 };
struct PtrWhere {
  int kind;     // PtrKind
  int device;   // the device ordinal of kPtrDevice / kPtrManaged memory
};

// The largest extents of a batch: level L (the weight and residual maps) and level 0 (the mask).
struct MapsExtent {
  int w, h, w0, h0;
};

// Why the outputs are refused, or "" if they are accepted; `device` is the context's device, where(const void*) -> PtrWhere.
// n <= 0 is left to the batch checks that follow.  Returns the message prefixed with "match_batch_maps: ".
template <typename Where>
std::string maps_args_error(const dvo_b200_weight_maps* m, int32_t n, const MapsExtent& e, int device, Where where) {
  const std::string fn = "match_batch_maps: ";
  if (!m) return fn + "maps is null";
  if (m->memory != DVO_B200_MAPS_DEVICE && m->memory != DVO_B200_MAPS_HOST) return fn + "unknown memory " + std::to_string(m->memory);
  if (!m->weight.data && !m->residual_i.data && !m->residual_z.data && !m->mask.data && !m->estimate && !m->precision)
    return fn + "no output requested";
  if (m->mask.data && !(std::isfinite(m->mask_weight) && m->mask_weight > 0.f)) return fn + "mask_weight must be finite and > 0";
  if (n <= 0) return "";
  // the first and last byte of [p, p + bytes) must lie where `memory` says
  auto placed = [&](const char* name, const void* p, int64_t bytes) -> std::string {
    const unsigned char* b = static_cast<const unsigned char*>(p);
    for (const void* q : {p, static_cast<const void*>(b + (bytes - 1))}) {
      const PtrWhere w = where(q);
      if (m->memory == DVO_B200_MAPS_DEVICE && !((w.kind == kPtrDevice || w.kind == kPtrManaged) && w.device == device))
        return fn + name + " is not device or managed memory of device " + std::to_string(device);
      if (m->memory == DVO_B200_MAPS_HOST && w.kind == kPtrDevice) return fn + name + " lies in device memory";
    }
    return "";
  };
  struct Plane { const char* name; const dvo_b200_map_plane* p; int64_t elem; int w, h; };
  const Plane planes[4] = {{"weight", &m->weight, 4, e.w, e.h}, {"residual_i", &m->residual_i, 4, e.w, e.h},
                           {"residual_z", &m->residual_z, 4, e.w, e.h}, {"mask", &m->mask, 1, e.w0, e.h0}};
  for (const Plane& q : planes) {
    if (!q.p->data) continue;
    const std::string name = q.name;
    const int64_t row = q.p->row_bytes, img = q.p->image_bytes;
    if (row < (int64_t)q.w * q.elem || row % q.elem != 0)
      return fn + name + ".row_bytes " + std::to_string(row) + " is below " + std::to_string(q.w) + " x " + std::to_string(q.elem) +
             " or not a multiple of " + std::to_string(q.elem);
    if (img / row < q.h) return fn + name + ".image_bytes " + std::to_string(img) + " is below " + std::to_string(q.h) + " rows";
    if (img % q.elem != 0 || (uintptr_t)q.p->data % (uintptr_t)q.elem != 0) return fn + name + " is misaligned";
    if (img > (INT64_MAX - row * q.h) / n) return fn + name + ".image_bytes is too large";
    const std::string why = placed(q.name, q.p->data, (int64_t)(n - 1) * img + (int64_t)(q.h - 1) * row + (int64_t)q.w * q.elem);
    if (!why.empty()) return why;
  }
  if (m->estimate) {
    if ((uintptr_t)m->estimate % sizeof(double) != 0) return fn + "estimate is misaligned";
    const std::string why = placed("estimate", m->estimate, (int64_t)n * 16 * (int64_t)sizeof(double));
    if (!why.empty()) return why;
  }
  if (m->precision) {
    if ((uintptr_t)m->precision % sizeof(float) != 0) return fn + "precision is misaligned";
    const std::string why = placed("precision", m->precision, (int64_t)n * 4 * (int64_t)sizeof(float));
    if (!why.empty()) return why;
  }
  return "";
}

}  // namespace dvo_b200
