// sharded.cu -- one-process multi-GPU front end of the C ABI (SURVEY.md 8b/8e): a batch of independent alignments is cut
// into contiguous shards of pair indices, one shard per device, each driven by its own context on its own host thread.
// This is the shape of the reference's callers: ConstraintProposalValidator::validate
// (dvo_slam/src/constraints/constraint_proposal_validator.cpp:141-146) and the TBB proposal search
// (dvo_slam/src/keyframe_graph.cpp:587-590) are single-process C++ loops over independent DenseTracker::match() calls.
// The alignments exchange nothing; the only "gather" is every shard writing its results into its own range of the caller's
// host array (device -> pinned host on the shard's stream), so a one-process caller needs no NCCL communicator.  The
// multi-process form of the same sharding (one rank per GPU, NCCL all-gather of the result records) is
// dvo_slam_b200/distributed.py on top of dvo_b200_match_batch_device.
//
// Written against the public C ABI only (include/dvo_b200.h): a caller could do the same with its own threads.  The checks
// and the slicing of dvo_b200_match_batch_modes_sharded are those of modes_args.h, which reads nothing but what the ABI
// exposes.
#include <cuda_runtime.h>

#include <string>
#include <thread>
#include <vector>

#include "../../include/dvo_b200.h"
#include "modes_args.h"

struct dvo_b200_sharded {
  std::vector<int> devices;
  std::vector<dvo_b200_ctx*> ctx;
  std::string last_error;
};

namespace {

int fail(dvo_b200_sharded* s, int code, const std::string& msg) {
  if (s) s->last_error = msg;
  return code;
}

// contiguous shard [begin, end) of `total` items for shard `k` of `n`: the remainder goes to the first shards (the same
// partition as dvo_slam_b200/distributed.py:shard_range, so one-process and multi-process runs own the same pairs)
void shard_range(int64_t total, int n, int k, int64_t* begin, int64_t* end) {
  const int64_t base = total / n, rem = total % n;
  *begin = k * base + (k < rem ? k : rem);
  *end = *begin + base + (k < rem ? 1 : 0);
}

template <typename F>
int for_each_shard(dvo_b200_sharded* s, int64_t total, F&& body) {
  const int n = int(s->ctx.size());
  std::vector<int> rc(size_t(n), 0);
  std::vector<std::thread> threads;
  for (int k = 0; k < n; ++k) {
    int64_t b, e;
    shard_range(total, n, k, &b, &e);
    if (b == e) continue;
    threads.emplace_back([&, k, b, e] { rc[size_t(k)] = body(k, b, e); });
  }
  for (std::thread& t : threads) t.join();
  for (int k = 0; k < n; ++k)
    if (rc[size_t(k)] != 0)
      return fail(s, rc[size_t(k)], "shard " + std::to_string(k) + " (device " + std::to_string(s->devices[size_t(k)]) + "): " +
                                        dvo_b200_last_error(s->ctx[size_t(k)]));
  return 0;
}

// What modes_args.h reads of a pyramid and of a pointer, through the public ABI and the CUDA runtime
dvo_b200::PyramidView public_view(const dvo_b200_pyramid* p, int level) {
  dvo_b200::PyramidView v{dvo_b200_pyramid_num_levels(p), dvo_b200_pyramid_device(p), 0, 0, 0, 0};
  dvo_b200_pyramid_level_info(p, 0, &v.w0, &v.h0, nullptr);
  dvo_b200_pyramid_level_info(p, level, &v.w, &v.h, nullptr);   // leaves 0 x 0 for a level the pyramid does not have
  return v;
}

dvo_b200::PtrWhere public_where(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return {dvo_b200::kPtrHost, -1}; }
  if (a.type == cudaMemoryTypeDevice) return {dvo_b200::kPtrDevice, a.device};
  if (a.type == cudaMemoryTypeManaged) return {dvo_b200::kPtrManaged, a.device};
  return {dvo_b200::kPtrHost, -1};
}

// E of a shard's slice (modes_args.h: modes_entry) on the shard's context
int call_entry(dvo_b200_ctx* ctx, const dvo_b200::ModesArgs& a) {
  switch (dvo_b200::modes_entry(a)) {
    case dvo_b200::kEntryMatch:
      return dvo_b200_match_batch(ctx, a.cfg, a.n, a.refs, a.curs, a.hypotheses, a.results, a.iter_stats, a.max_log);
    case dvo_b200::kEntryPhotometric:
      return dvo_b200_match_batch_photometric(ctx, a.cfg, a.n, a.refs, a.curs, a.hypotheses, a.ab_init, a.results, a.ab, a.iter_stats,
                                              a.max_log);
    case dvo_b200::kEntryPrior:
      return dvo_b200_match_batch_prior(ctx, a.cfg, a.n, a.refs, a.curs, a.hypotheses, a.prior, a.ab_init, a.ab, a.results, a.iter_stats,
                                        a.max_log);
    case dvo_b200::kEntryMaps:
      return dvo_b200_match_batch_maps(ctx, a.cfg, a.n, a.refs, a.curs, a.hypotheses, a.prior, a.ab_init, a.ab, a.results, a.iter_stats,
                                       a.max_log, a.maps);
    case dvo_b200::kEntryHypotheses:
      break;
  }
  return dvo_b200_match_batch_hypotheses_modes(ctx, a.cfg, a.n, a.refs, a.curs, a.k, a.hypotheses, a.screen_level, a.min_ratio, a.prior,
                                               a.ab_init, a.ab, a.screen_ab, a.results, a.best, a.scores, a.screen_results, a.iter_stats,
                                               a.max_log, a.maps);
}

}  // namespace

extern "C" {

int dvo_b200_sharded_create(int32_t n_devices, const int32_t* devices, dvo_b200_sharded** out) {
  if (!out || n_devices < 1) return DVO_B200_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  dvo_b200_sharded* s = new dvo_b200_sharded;
  for (int k = 0; k < n_devices; ++k) {
    const int dev = devices ? devices[k] : k;
    dvo_b200_ctx* c = nullptr;
    const int rc = dvo_b200_create(dev, nullptr, &c);   // fails loudly without a usable device: there is no CPU path
    if (rc != 0) {
      for (dvo_b200_ctx* q : s->ctx) dvo_b200_destroy(q);
      delete s;
      return rc;
    }
    s->devices.push_back(dev);
    s->ctx.push_back(c);
  }
  *out = s;
  return 0;
}

int dvo_b200_sharded_destroy(dvo_b200_sharded* s) {
  if (!s) return DVO_B200_ERR_INVALID_ARGUMENT;
  for (dvo_b200_ctx* c : s->ctx) dvo_b200_destroy(c);
  delete s;
  return 0;
}

int32_t dvo_b200_sharded_num_shards(const dvo_b200_sharded* s) { return s ? int32_t(s->ctx.size()) : 0; }

dvo_b200_ctx* dvo_b200_sharded_ctx(dvo_b200_sharded* s, int32_t shard) {
  return (s && shard >= 0 && size_t(shard) < s->ctx.size()) ? s->ctx[size_t(shard)] : nullptr;
}

const char* dvo_b200_sharded_last_error(dvo_b200_sharded* s) { return s ? s->last_error.c_str() : "null sharded handle"; }

int dvo_b200_shard_range(int64_t total, int32_t n_shards, int32_t shard, int64_t* begin, int64_t* end) {
  if (total < 0 || n_shards < 1 || shard < 0 || shard >= n_shards || !begin || !end) return DVO_B200_ERR_INVALID_ARGUMENT;
  shard_range(total, n_shards, shard, begin, end);
  return 0;
}

int dvo_b200_sharded_pyramid_create_batch(dvo_b200_sharded* s, int32_t n, const float* intensity, const float* depth, int32_t width,
                                          int32_t height, float fx, float fy, float ox, float oy, int32_t levels,
                                          dvo_b200_pyramid** out) {
  if (!s || n < 1 || !intensity || !depth || !out) return fail(s, DVO_B200_ERR_INVALID_ARGUMENT, "sharded_pyramid_create_batch: bad argument");
  const size_t npx = size_t(width) * size_t(height);
  int rc = for_each_shard(s, n, [&](int k, int64_t b, int64_t e) {
    int r = dvo_b200_pyramid_create_batch(s->ctx[size_t(k)], int32_t(e - b), intensity + size_t(b) * npx, depth + size_t(b) * npx, width, height,
                                          fx, fy, ox, oy, levels, out + b);
    return r != 0 ? r : dvo_b200_synchronize(s->ctx[size_t(k)]);   // the host images may be released on return
  });
  return rc;
}

int dvo_b200_sharded_pyramid_create_raw_batch(dvo_b200_sharded* s, int32_t n, const uint8_t* grey, const uint16_t* raw_depth,
                                              float depth_scale, int32_t width, int32_t height, float fx, float fy, float ox, float oy,
                                              int32_t levels, dvo_b200_pyramid** out) {
  if (!s || n < 1 || !grey || !raw_depth || !out) return fail(s, DVO_B200_ERR_INVALID_ARGUMENT, "sharded_pyramid_create_raw_batch: bad argument");
  const size_t npx = size_t(width) * size_t(height);
  return for_each_shard(s, n, [&](int k, int64_t b, int64_t e) {
    int r = dvo_b200_pyramid_create_raw_batch(s->ctx[size_t(k)], int32_t(e - b), grey + size_t(b) * npx, raw_depth + size_t(b) * npx, depth_scale,
                                              width, height, fx, fy, ox, oy, levels, out + b);
    return r != 0 ? r : dvo_b200_synchronize(s->ctx[size_t(k)]);
  });
}

int dvo_b200_match_batch_sharded(dvo_b200_sharded* s, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                                 dvo_b200_pyramid* const* currents, const double* T_init, dvo_b200_result* results,
                                 dvo_b200_iteration_stats* iteration_stats, int32_t max_iteration_stats) {
  if (!s || !cfg || n < 1 || !references || !currents || !results) return fail(s, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_sharded: bad argument");
  const int ns = int(s->ctx.size());
  for (int k = 0; k < ns; ++k) {   // every pair must already live on the device of the shard that owns its index
    int64_t b, e;
    shard_range(n, ns, k, &b, &e);
    for (int64_t i = b; i < e; ++i) {
      const int dr = dvo_b200_pyramid_device(references[i]), dc = dvo_b200_pyramid_device(currents[i]);
      if (dr != s->devices[size_t(k)] || dc != s->devices[size_t(k)])
        return fail(s, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_sharded: pair " + std::to_string(i) + " belongs to shard " + std::to_string(k) +
                                                          " (device " + std::to_string(s->devices[size_t(k)]) + ") but its pyramids live on devices " +
                                                          std::to_string(dr) + " / " + std::to_string(dc));
    }
  }
  return for_each_shard(s, n, [&](int k, int64_t b, int64_t e) {
    return dvo_b200_match_batch(s->ctx[size_t(k)], cfg, int32_t(e - b), references + b, currents + b, T_init ? T_init + 16 * b : nullptr, results + b,
                                iteration_stats ? iteration_stats + size_t(b) * size_t(max_iteration_stats) : nullptr, max_iteration_stats);
  });
}

int dvo_b200_match_batch_modes_sharded(dvo_b200_sharded* s, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                                       dvo_b200_pyramid* const* currents, int32_t k, const double* hypotheses, int32_t screen_level,
                                       double min_constraint_ratio, const double* prior_information, const double* photometric_init,
                                       double* photometric, double* screen_photometric, dvo_b200_result* results, int32_t* best,
                                       double* scores, dvo_b200_result* screen_results, dvo_b200_iteration_stats* iteration_stats,
                                       int32_t max_iteration_stats, const dvo_b200_weight_maps* maps) {
  if (!s) return DVO_B200_ERR_INVALID_ARGUMENT;
  dvo_b200::ModesArgs a;
  a.cfg = cfg; a.n = n; a.refs = references; a.curs = currents; a.k = k; a.hypotheses = hypotheses; a.screen_level = screen_level;
  a.min_ratio = min_constraint_ratio; a.prior = prior_information; a.ab_init = photometric_init; a.ab = photometric;
  a.screen_ab = screen_photometric; a.results = results; a.best = best; a.scores = scores; a.screen_results = screen_results;
  a.iter_stats = iteration_stats; a.max_log = max_iteration_stats; a.maps = maps;
  // the whole batch is checked before any shard starts, so a refusal leaves every shard's context untouched
  int code = 0;
  const std::string why = dvo_b200::modes_args_error(a, dvo_b200::kFormSharded, int(s->ctx.size()), s->devices.data(), public_view,
                                                     public_where, &code);
  if (!why.empty()) return fail(s, code, why);
  return for_each_shard(s, n, [&](int shard, int64_t b, int64_t e) {
    dvo_b200_weight_maps m;
    return call_entry(s->ctx[size_t(shard)], dvo_b200::shard_slice(a, b, e, &m));
  });
}

}  // extern "C"
