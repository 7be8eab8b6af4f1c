// modes_args.h -- dvo_b200_match_batch_modes_device and dvo_b200_match_batch_modes_sharded: which existing entry point E a set
// of arguments stands for, every check made before anything is staged or launched (E's own, in E's order, then those of the
// form), and the slice of a batch that one shard runs.  Plain C++ without CUDA, so that they can be built and run on the
// host alone (tests/native/modes_args.cpp): where a pointer lies is asked through `where` (maps_args.h) and what a pyramid
// is through `view`, which capi.cu answers from the pyramid's fields, sharded.cu through the public ABI and the host test
// with fakes.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <string>

#include "../../include/dvo_b200.h"
#include "hypotheses_args.h"
#include "maps_args.h"
#include "prior_args.h"

namespace dvo_b200 {

// The arguments of the two forms, in their order.  k = 0: one plain alignment per pair, `hypotheses` is T_init (n * 16 or
// NULL), prior n * 36 and ab_init 2n; k >= 1: the layouts of dvo_b200_match_batch_hypotheses_modes.
struct ModesArgs {
  const dvo_b200_config* cfg = nullptr;
  int32_t n = 0;
  dvo_b200_pyramid* const* refs = nullptr;
  dvo_b200_pyramid* const* curs = nullptr;
  int32_t k = 0;
  const double* hypotheses = nullptr;
  int32_t screen_level = 0;
  double min_ratio = 0.0;
  const double* prior = nullptr;
  const double* ab_init = nullptr;
  double* ab = nullptr;
  double* screen_ab = nullptr;
  dvo_b200_result* results = nullptr;
  int32_t* best = nullptr;
  double* scores = nullptr;
  dvo_b200_result* screen_results = nullptr;
  dvo_b200_iteration_stats* iter_stats = nullptr;
  int32_t max_log = 0;
  const dvo_b200_weight_maps* maps = nullptr;
};

// E: k >= 1 dvo_b200_match_batch_hypotheses_modes; k = 0 by what is non-NULL: maps -> dvo_b200_match_batch_maps, else
// prior -> _prior, else photometric -> _photometric, else dvo_b200_match_batch.
enum ModesEntry { kEntryMatch, kEntryPhotometric, kEntryPrior, kEntryMaps, kEntryHypotheses };
inline ModesEntry modes_entry(const ModesArgs& a) {
  if (a.k != 0) return kEntryHypotheses;
  if (a.maps) return kEntryMaps;
  if (a.prior) return kEntryPrior;
  return a.ab ? kEntryPhotometric : kEntryMatch;
}

// What the checks read of one pyramid: its level count and device, the size of level 0 and of the level asked for (0 x 0
// if it has no such level).
struct PyramidView {
  int levels, device, w0, h0, w, h;
};

// The largest extents of a batch's references at cfg->last_level and level 0, or false for a batch the match would refuse
// (the maps are then checked as for n = 0 and the batch checks refuse it).  view(p, level) -> PyramidView.
template <typename View>
bool batch_maps_extent(const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* refs, View view, MapsExtent* ext) {
  *ext = MapsExtent{0, 0, 0, 0};
  if (!(cfg && n > 0 && refs && cfg->last_level >= 0 && cfg->last_level < DVO_B200_MAX_LEVELS)) return false;
  for (int32_t i = 0; i < n; ++i) {
    if (!refs[i]) return false;
    const PyramidView r = view(refs[i], cfg->last_level);
    if (r.levels <= cfg->last_level) return false;
    ext->w = std::max(ext->w, r.w); ext->h = std::max(ext->h, r.h);
    ext->w0 = std::max(ext->w0, r.w0); ext->h0 = std::max(ext->h0, r.h0);
  }
  return true;
}

// The batch checks every match makes (tracker.cu: check_batch), in its order; *code is the status of the refusal.
template <typename View>
std::string batch_args_error(const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* refs, dvo_b200_pyramid* const* curs,
                             View view, int* code) {
  *code = DVO_B200_ERR_INVALID_ARGUMENT;
  if (!cfg || n <= 0 || !refs || !curs) return "match: null argument";
  if (cfg->first_level < cfg->last_level || cfg->last_level < 0 || cfg->first_level >= DVO_B200_MAX_LEVELS)
    return "match: config not sane (FirstLevel >= LastLevel >= 0 required)";
  if (cfg->max_iterations_per_level < 0) return "match: max iterations < 0";
  PyramidView first{};
  for (int32_t i = 0; i < n; ++i) {
    if (!refs[i] || !curs[i]) return "match: null pyramid";
    const PyramidView r = view(refs[i], 0), c = view(curs[i], 0);
    if (i == 0) first = r;
    if (r.levels <= cfg->first_level || c.levels <= cfg->first_level) return "match: pyramid has fewer levels than FirstLevel+1";
    if (r.w0 != first.w0 || r.h0 != first.h0 || c.w0 != first.w0 || c.h0 != first.h0) {
      *code = DVO_B200_ERR_SHAPE_MISMATCH;
      return "match: all pyramids of a batch must share width/height";
    }
  }
  return "";
}

inline bool finite_rows(const double* v, size_t count) {
  for (size_t i = 0; i < count; ++i)
    if (!std::isfinite(v[i])) return false;
  return true;
}

// The argument checks of E before its batch checks, in E's order and with E's messages (capi.cu: the entry points).  ext:
// the batch's extents, or NULL for a batch the match would refuse; device: the context's device, for maps in device memory.
template <typename Where>
std::string entry_args_error(ModesEntry e, const ModesArgs& a, const MapsExtent* ext, int device, Where where) {
  const size_t ab_rows = 2 * (size_t)(a.n > 0 ? a.n : 0);
  switch (e) {
    case kEntryMatch:
      return a.results ? "" : "match_batch: null argument";
    case kEntryPhotometric:
      if (!a.results || !a.ab) return "match_batch_photometric: null argument";
      if (a.ab_init && !finite_rows(a.ab_init, ab_rows)) return "match_batch_photometric: photometric_init is not finite";
      return "";
    case kEntryPrior: {
      if (!a.results) return "match_batch_prior: null argument";
      const std::string why = prior_args_error(a.cfg, a.n, a.prior, a.ab_init, a.ab);
      if (!why.empty()) return why;
      if (a.ab_init && !finite_rows(a.ab_init, ab_rows)) return "match_batch_prior: photometric_init is not finite";
      return "";
    }
    case kEntryMaps: {
      if (!a.results) return "match_batch_maps: null argument";
      if (a.prior) {
        const std::string why = prior_args_error(a.cfg, a.n, a.prior, a.ab_init, a.ab);
        if (!why.empty()) return why;
      } else if (a.ab_init && !a.ab) {
        return "match_batch_maps: photometric_init without photometric";
      }
      if (a.ab_init && !finite_rows(a.ab_init, ab_rows)) return "match_batch_maps: photometric_init is not finite";
      return maps_args_error(a.maps, ext ? a.n : 0, ext ? *ext : MapsExtent{0, 0, 0, 0}, device, where);
    }
    case kEntryHypotheses:
      return hypotheses_modes_args_error(a.cfg, a.n, a.k, a.hypotheses, a.screen_level, a.min_ratio, a.results, a.best, a.prior,
                                         a.ab_init, a.ab, a.screen_ab, a.maps, ext, device, where);
  }
  return "";
}

// The two forms of the call
enum ModesForm { kFormDevice, kFormSharded };

inline const char* form_name(ModesForm f) { return f == kFormDevice ? "match_batch_modes_device: " : "match_batch_modes_sharded: "; }

// One output of the call: its name, pointer, bytes for the whole batch and element alignment (bytes 0: not passed)
struct ModesOutput {
  const char* name;
  const void* p;
  int64_t bytes, align;
};

// The outputs of a call other than the maps, in argument order
inline void modes_outputs(const ModesArgs& a, ModesOutput out[7]) {
  const int64_t n = a.n, nk = (int64_t)a.n * a.k, logs = a.iter_stats && a.max_log > 0 ? a.max_log : 0;
  out[0] = {"photometric", a.ab, 2 * n * (int64_t)sizeof(double), (int64_t)sizeof(double)};
  out[1] = {"screen_photometric", a.screen_ab, 2 * nk * (int64_t)sizeof(double), (int64_t)sizeof(double)};
  out[2] = {"results", a.results, n * (int64_t)sizeof(dvo_b200_result), (int64_t)alignof(dvo_b200_result)};
  out[3] = {"best", a.best, n * (int64_t)sizeof(int32_t), (int64_t)sizeof(int32_t)};
  out[4] = {"scores", a.scores, nk * (int64_t)sizeof(double), (int64_t)sizeof(double)};
  out[5] = {"screen_results", a.screen_results, nk * (int64_t)sizeof(dvo_b200_result), (int64_t)alignof(dvo_b200_result)};
  out[6] = {"iteration_stats", logs ? a.iter_stats : nullptr, n * logs * (int64_t)sizeof(dvo_b200_iteration_stats),
            (int64_t)alignof(dvo_b200_iteration_stats)};
}

// Every check of dvo_b200_match_batch_modes_device (form kFormDevice, ndev = 1, devices = the context's device) or
// _modes_sharded (kFormSharded, the shards' devices), in this order:
//   1. everything E refuses before its batch checks (entry_args_error; maps placed as on devices[0]);
//   2. E's batch checks (batch_args_error, over the whole batch);
//   3. k = 0: an output that only k >= 1 writes (best, scores, screen_results, screen_photometric), or photometric_init
//      without photometric;
//   4. device: maps in DVO_B200_MAPS_HOST; then per output in argument order, a misaligned pointer, and a first or last byte
//      that `where` does not report as device or managed memory of the context's device;
//      sharded: per pair, pyramids off the device of the shard that owns the pair (dvo_b200_shard_range); then maps in
//      DVO_B200_MAPS_DEVICE.
// Returns "" or the message; *code is the status to return (DVO_B200_ERR_SHAPE_MISMATCH for a batch of mixed sizes, else
// DVO_B200_ERR_INVALID_ARGUMENT).  The messages of 1 and 2 are E's own; those of 3 and 4 start with the form's name.
template <typename View, typename Where>
std::string modes_args_error(const ModesArgs& a, ModesForm form, int ndev, const int* devices, View view, Where where, int* code) {
  *code = DVO_B200_ERR_INVALID_ARGUMENT;
  MapsExtent ext;
  const bool sane = a.maps && batch_maps_extent(a.cfg, a.n, a.refs, view, &ext);
  std::string why = entry_args_error(modes_entry(a), a, sane ? &ext : nullptr, devices[0], where);
  if (!why.empty()) return why;
  why = batch_args_error(a.cfg, a.n, a.refs, a.curs, view, code);
  if (!why.empty()) return why;
  const std::string fn = form_name(form);
  if (a.k == 0) {
    const struct { const char* name; const void* p; } only_k[4] = {
        {"best", a.best}, {"scores", a.scores}, {"screen_results", a.screen_results}, {"screen_photometric", a.screen_ab}};
    for (const auto& o : only_k)
      if (o.p) return fn + o.name + " is only written with k >= 1";
    if (a.ab_init && !a.ab) return fn + "photometric_init without photometric";
  }
  if (form == kFormDevice) {
    if (a.maps && a.maps->memory == DVO_B200_MAPS_HOST) return fn + "maps must be DVO_B200_MAPS_DEVICE";
    ModesOutput out[7];
    modes_outputs(a, out);
    for (const ModesOutput& o : out) {
      if (!o.p || o.bytes <= 0) continue;
      if ((uintptr_t)o.p % (uintptr_t)o.align != 0) return fn + o.name + " is misaligned";
      const unsigned char* b = static_cast<const unsigned char*>(o.p);
      for (const void* q : {o.p, static_cast<const void*>(b + (o.bytes - 1))}) {
        const PtrWhere w = where(q);
        if (!((w.kind == kPtrDevice || w.kind == kPtrManaged) && w.device == devices[0]))
          return fn + o.name + " is not device or managed memory of device " + std::to_string(devices[0]);
      }
    }
    return "";
  }
  for (int s = 0; s < ndev; ++s) {
    const int64_t base = a.n / ndev, rem = a.n % ndev;   // dvo_b200_shard_range
    const int64_t b = s * base + (s < rem ? s : rem), e = b + base + (s < rem ? 1 : 0);
    for (int64_t i = b; i < e; ++i) {
      const int dr = view(a.refs[i], 0).device, dc = view(a.curs[i], 0).device;
      if (dr != devices[s] || dc != devices[s])
        return fn + "pair " + std::to_string(i) + " belongs to shard " + std::to_string(s) + " (device " + std::to_string(devices[s]) +
               ") but its pyramids live on devices " + std::to_string(dr) + " / " + std::to_string(dc);
    }
  }
  if (a.maps && a.maps->memory == DVO_B200_MAPS_DEVICE) return fn + "maps must be DVO_B200_MAPS_HOST";
  return "";
}

// The arguments of pairs [b, e) of a: every per-pair input and output at that pair's offset (k of them per pair where the
// layout is per hypothesis, max_log iteration-log entries per pair), the maps' planes at data + b * image_bytes and their
// estimate and precision at pair b.  `maps` receives the sliced description (a.maps NULL: unused).
inline ModesArgs shard_slice(const ModesArgs& a, int64_t b, int64_t e, dvo_b200_weight_maps* maps) {
  ModesArgs s = a;
  const int64_t per = a.k ? a.k : 1;   // rows of a per-pair input
  auto at = [&](auto* p, int64_t stride) { return p ? p + b * stride : p; };
  s.n = (int32_t)(e - b);
  s.refs = a.refs + b;
  s.curs = a.curs + b;
  s.hypotheses = at(a.hypotheses, 16 * per);
  s.prior = at(a.prior, 36 * per);
  s.ab_init = at(a.ab_init, 2 * per);
  s.ab = at(a.ab, 2);
  s.screen_ab = at(a.screen_ab, 2 * (int64_t)a.k);
  s.results = at(a.results, 1);
  s.best = at(a.best, 1);
  s.scores = at(a.scores, (int64_t)a.k);
  s.screen_results = at(a.screen_results, (int64_t)a.k);
  s.iter_stats = at(a.iter_stats, (int64_t)std::max(a.max_log, 0));
  if (a.maps) {
    *maps = *a.maps;
    for (dvo_b200_map_plane* q : {&maps->weight, &maps->residual_i, &maps->residual_z, &maps->mask})
      if (q->data) q->data = static_cast<char*>(q->data) + b * q->image_bytes;
    maps->estimate = at(maps->estimate, 16);
    maps->precision = at(maps->precision, 4);
    s.maps = maps;
  }
  return s;
}

}  // namespace dvo_b200
