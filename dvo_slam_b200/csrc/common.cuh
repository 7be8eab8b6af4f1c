// common.cuh -- host/device data model shared by the pyramid and tracker translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/dvo_b200.h"
#include "create_args.h"
#include "modes_args.h"
#include "se3.cuh"

namespace dvo_b200 {

// Unusable-pixel summary of one level of a pyramid whose mask also acts in the CURRENT role: a summed-area table of the
// unusable pixel counts over kSatBlock x kSatBlock blocks, (ceil(w/8) + 1) x (ceil(h/8) + 1) ints, row 0 and column 0 zero.
// Whether a rectangle of the level holds an unusable pixel is then four loads (a conservative answer at block granularity).
constexpr int kSatBlock = 8;
__host__ __device__ __forceinline__ int sat_cols(int w) { return (w + kSatBlock - 1) / kSatBlock + 1; }
__host__ __device__ __forceinline__ int sat_rows(int h) { return (h + kSatBlock - 1) / kSatBlock + 1; }

// Reference tile record: everything the level kernel reads of the REFERENCE image for one tile, contiguous in HBM so that
// one bulk copy stages it (row-major planes cost one copy per tile row and plane: 14 of the ~29 copies of a stage-B tile):
//   kTileH rows x kTileW of (I, Zsel)   Zsel = depth where the pixel is a selected reference point, NaN elsewhere
//   kTileW floats tx                     point-cloud template of the tile's columns
//   kTileH rows x kTileW of (Ix, Iy)     only stage B copies this part
// Cells outside the image hold (0, NaN) / 0 / (0, 0).
constexpr int kRecTx = kTileH * kTileW;              // float2 offset of tx[]
constexpr int kRecP1 = kRecTx + kTileW / 2;          // float2 offset of the gradient rows
constexpr int kRecF2 = kRecP1 + kTileH * kTileW;     // float2 elements per record (18 560 bytes)
// the bulk copies of a record (whole, or up to kRecP1 in stage A) need 16-byte multiples, and so do record offsets in HBM
static_assert(kTileW % 32 == 0 && (kRecP1 * 8) % 16 == 0 && (kRecF2 * 8) % 16 == 0, "tile records must stay 16-byte granular");
__host__ __device__ __forceinline__ size_t rec_cell(int x, int y, int nbands) {   // (I, Zsel) of pixel (x, y) relative to the level's records
  return (size_t)((y / kTileH) * nbands + x / kTileW) * kRecF2 + (size_t)(y % kTileH) * kTileW + (x % kTileW);
}

struct Slab;
// Pool of released slabs of one context, keyed by size (release -> reuse instead of cudaFree).  Pyramids are
// independent objects in the reference (boost::shared_ptr<RgbdImagePyramid>) and routinely outlive the tracker that
// first used them, and they may be released from another host thread than the one that built them: the pool is
// shared-owned by the context and by every slab, and guarded by its own mutex.
struct SlabPool {
  std::mutex mu;
  std::multimap<size_t, Slab*> free;
  bool closed = false;           // the context is gone: released slabs are freed instead of pooled
  int device = 0;
};

struct Slab {                  // one cudaMalloc shared by a batch of pyramids
  void* base = nullptr;
  size_t bytes = 0;
  int refs = 0;
  cudaEvent_t ready = nullptr;   // recorded on the creating stream after the build kernels (and after a re-selection)
  // Work of OTHER contexts that may still read the slab: per consuming context (dvo_b200_ctx::uid), one event recorded
  // on its stream after its latest call that read the slab.  Guarded by pool->mu.  A pyramid may be released as soon as
  // such a call has returned, so the owner's next build into this slab (acquire_slab) waits for these events first.
  std::vector<std::pair<uint64_t, cudaEvent_t>> foreign_uses;
  std::shared_ptr<SlabPool> pool;
};

// Sets the calling thread's current device for a scope and restores the previous one: for the calls that need no context
// (download with a NULL context, the last release of a pyramid) and so must not change the caller's device.
struct DeviceScope {
  int prev = -1;
  explicit DeviceScope(int device) {
    if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
    if (prev != device) cudaSetDevice(device);
  }
  ~DeviceScope() { if (prev >= 0) cudaSetDevice(prev); }
};

}  // namespace dvo_b200

// opaque handle types of the C ABI
struct dvo_b200_pyramid {
  dvo_b200_ctx* ctx = nullptr;   // the context that built it (may be gone by the time the pyramid is read: never dereferenced for that)
  int device = 0;                // CUDA ordinal the planes live on
  std::atomic<int> refcount{1};   // retain/release may come from any host thread (boost::shared_ptr semantics)
  int levels = 0;
  dvo_b200::LevelInfo L[dvo_b200::kMaxLevels];
  dvo_b200::Slab* slab = nullptr;
  float2* planes = nullptr;      // device
  uint32_t* sel_mask = nullptr;  // device: selection bitmasks of all levels (default thresholds)
  int* sel_info = nullptr;       // device: per level {S, last selected linear pixel index}
  float* tmpl = nullptr;         // device: per level tx[w], ty[h] point-cloud template (rgbd_image.cpp:197-198)
  float2* tile_range = nullptr;  // device: per level, per tile {min, max} of the non-NaN Z' (min > max: none); of usable pixels only if masked
  uint32_t* usable = nullptr;    // device: per level usable bits of the reference mask, layout of sel_mask (NULL: built without a mask)
  int* cur_sat = nullptr;        // device: per level unusable-pixel summary (see kSatBlock); only if the mask acts in the current role
  int mask_roles = 0;            // 0: no mask; DVO_B200_MASK_ROLE_REFERENCE, optionally | DVO_B200_MASK_ROLE_CURRENT
  float sel_ti = 0.f, sel_td = 0.f;  // thresholds the masks were built with
  std::mutex sel_mu;                 // guards sel_ti / sel_td and the enqueueing of a re-selection
  uint64_t id = 0;
};

namespace dvo_b200 {

// ---- per-pair device state ---------------------------------------------------------------------
struct PairLevel {              // what one alignment reads at the current level (uploaded per level)
  const float2* r0;                    // reference tile records of the level
  const float2* rp0;                   // the reference's own P0 = (I, Z') plane (corrected estimator: depth of the odd last point)
  const uint32_t* rmask;               // reference selection mask
  const int* rsel;                     // {S, last selected pixel}
  const float* rtmpl;                  // tx[w], ty[h]
  const float2* rrange;                // per-tile depth range of the reference
  const float2* c0; const float2* c3;  // current P0 (I, Z') and P2 (I, Z)
  float cfx, cfy, cox, coy;            // current-image intrinsics (dense_tracking.cpp:212)
  long long max_valid_pixels;          // PointSelection::getMaximumNumberOfPoints
};
// What a pair reads at the current level in the level kernel instance with current-role masks (tracker.cu, kCurMask).  The
// summary pointer travels in an array of its own (Workspace::d_csat, same index as the descriptors): PairLevel is copied
// to the stack of the level kernel, and a bigger PairLevel would change the stack frame of the default instances.
struct CurPairLevel : PairLevel {
  const int* csat;                     // unusable-pixel summary of the current image's level (NULL: no mask in the current role)
};

struct LevelSummary {           // device mirror of dvo_b200_level_stats
  int id, termination;
  long long max_valid_pixels, valid_pixels;
  int num_iterations, has_inc;
  long long last_n, last_inc_n;
  double last_inc_nll;
};

struct PairState {
  SE3d estimate, estimate_old, initial, initial_old, inc;   // Revertable<SE3d> (util/revertable.h:45-55)
  double x[6];                  // current increment
  double error, last_error;     // IterationContext::Error / LastError
  double A[36], b[6];           // last linearisation (A without mu)
  double A_done[36];            // EstimateInformation of the last completed iteration on this level (incl. mu)
  double nll_done, prior_done;  // its TDistributionLogLikelihood / PriorLogLikelihood
  double nll_cur, prior_cur;
  int have_done;
  float precision[4];           // P_k (row-major), also P_{k-1} on entry of an iteration
  float precision_prev[4];      // P_{k-1}: what the weights of the current iteration were computed with
  float ll;
  float kt[12];                 // K * float(estimate)[0:3,:]  (dense_tracking_impl.cpp:142-152)
  long long n;                  // valid constraints of the current iteration
  long long n_keep;             // 50*floor(n/50): log-likelihood terms kept (dense_tracking_impl.cpp:413-422)
  int iteration;                // IterationContext::Iteration
  int level_active;             // 1 while this pair still iterates on the current level
  int phase_ok;                 // 1 if the residual stage produced >= 6 constraints (normal stage runs)
  int termination;
  int num_levels;
  int num_iterations_total;
  int iter_log_count;
  int pad_;
  LevelSummary levels[kMaxLevels];

  // the Result is defined (not NaN): the last level has an accepted iteration (SURVEY Q24)
  __host__ __device__ bool result_defined() const {
    return have_done == 1 && termination != DVO_B200_TERM_TOO_FEW_CONSTRAINTS;
  }
};

// K * float(T)[0:3,:] in float, in the reference's operation order (dense_tracking_impl.cpp:142-152): every copy of K T must
// round alike (the weight maps recompute the level kernel's, DESIGN §4.10).
__device__ __forceinline__ void kt_of(const double T[16], const PairLevel& pl, float kt[12]) {
  for (int j = 0; j < 4; ++j) {
    const float t0 = (float)T[j], t1 = (float)T[4 + j], t2 = (float)T[8 + j];
    kt[j] = __fadd_rn(__fmul_rn(pl.cfx, t0), __fmul_rn(pl.cox, t2));
    kt[4 + j] = __fadd_rn(__fmul_rn(pl.cfy, t1), __fmul_rn(pl.coy, t2));
    kt[8 + j] = t2;
  }
}

// The affine brightness model of one pair (photometric alignments only: an array of its own, so that PairState and the
// default instances of the level kernel stay as they are).  (alpha, beta) is what the current iteration's residuals use
// (as float); old is the Revertable copy, restored together with the pose.  A / b: the 8 x 8 linearisation (no prior), written
// only for the linearisation hook.
struct AffineState {
  double ab[2], ab_old[2];
  double A[64], b[8];
};

struct Workspace {              // per-ctx scratch of the level kernel
  PairLevel* d_pair_level = nullptr; // one descriptor of slack past the last: k_stage_words copies whole 16-byte words
  const int** d_csat = nullptr;      // per descriptor of d_pair_level: CurPairLevel::csat (only written for kCurMask launches)
  PairState* d_state = nullptr;
  char* d_scratch = nullptr;         // the level kernel's per-launch scratch (tracker.cu: ScratchLayout)
  float* d_dump = nullptr;           // test hook: seven residual-record planes of one level
  double* d_tinit = nullptr;         // per pair initial estimate (4x4)
  dvo_b200_iteration_stats* d_iter_log = nullptr;
  AffineState* d_affine = nullptr;   // per pair of a photometric alignment
  double* d_prior = nullptr;         // per pair of an alignment with a motion prior: the 6 x 6 information, row-major
  char* d_maps = nullptr;            // weight maps copied back to the host (DVO_B200_MAPS_HOST): the kernel's packed output
  int* h_active = nullptr;           // pinned: per launch of a call, the kernel's error flag
  size_t cap_pair_level = 0, cap_state = 0, cap_scratch = 0, cap_iter_log = 0, cap_dump = 0, cap_tinit = 0, cap_csat = 0,
         cap_affine = 0, cap_prior = 0, cap_maps = 0;   // in elements (see grow)
};

}  // namespace dvo_b200

struct dvo_b200_ctx {
  int device = 0;
  uint64_t uid = 0;                   // unique over the process lifetime (a context's address may be reused after destroy)
  int num_sms = 0;                        // persistent-kernel grid geometry (queried once)
  int ctas_per_sm[2][2] = {{0, 0}, {0, 0}};   // [photometric][motion prior]: resident CTAs of those level kernel instances, 0 = not queried yet
  int estimator = DVO_B200_ESTIMATOR_REFERENCE;   // dvo_b200_estimator of every later alignment / test hook on this context
  unsigned long long* d_dbg = nullptr;   // DVO_B200_TIMING=1: per-level phase timers of the persistent kernel (64 slots)
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  std::string last_error;
  int64_t launches = 0, h2d_bytes = 0, d2h_bytes = 0;
  int pending_level_flags = 0;          // levels whose error flag has been copied to pinned memory but not yet checked
  uint64_t next_pyramid_id = 1;
  dvo_b200::Workspace ws;
  std::shared_ptr<dvo_b200::SlabPool> pool;   // pooled device slabs (see SlabPool)
  // staging for uploads
  void* d_stage = nullptr; size_t d_stage_bytes = 0;
  void* h_stage = nullptr; size_t h_stage_bytes = 0;   // pinned bounce buffer for pageable sources
  void* h_results = nullptr; size_t h_results_bytes = 0;  // pinned
  // profiling
  bool profile = false;
  double prof_ms[16] = {0};           // classes 0..7 (dvo_b200_profile_read); 8 + i: level kernel of the i-th level of a match
  int64_t prof_launches[16] = {0};
  std::vector<std::pair<int, std::pair<cudaEvent_t, cudaEvent_t>>> prof_pending;
  std::vector<cudaEvent_t> event_pool;
  std::mutex mu;
};

namespace dvo_b200 {

int set_error(dvo_b200_ctx* ctx, int code, const std::string& msg);
int check_cuda(dvo_b200_ctx* ctx, cudaError_t e, const char* what);

#define DVO_CUDA(ctx, call)                                              \
  do {                                                                   \
    int rc__ = ::dvo_b200::check_cuda((ctx), (call), #call);             \
    if (rc__ != 0) return rc__;                                          \
  } while (0)

// A workspace buffer of at least `need` elements: a smaller one is freed once the stream has drained, and the new one is
// uninitialised.
template <typename T>
int grow(dvo_b200_ctx* ctx, T*& ptr, size_t& cap, size_t need) {
  if (need <= cap) return 0;
  if (ptr) { cudaStreamSynchronize(ctx->stream); cudaFree(ptr); ptr = nullptr; cap = 0; }
  DVO_CUDA(ctx, cudaMalloc((void**)&ptr, need * sizeof(T)));
  cap = need;
  return 0;
}

// profiling scope: records start/stop events around a kernel class when enabled
struct ProfScope {
  dvo_b200_ctx* ctx; int cls; cudaEvent_t a = nullptr, b = nullptr;
  ProfScope(dvo_b200_ctx* c, int cls_, int nlaunch = 1);
  ~ProfScope();
};

// One plane of level-0 input in device memory: element (img, y, x) of the plane is data[img * stride + y * pitch + x], in
// elements of the plane's type (a pixel of interleaved BGR is 3 elements).  Packed planes: pitch = row elements, stride =
// pitch * h.  stride = 0: every image reads the same plane.
struct SrcPlane {
  const void* data;
  int64_t pitch, stride;
  __host__ __device__ size_t at(int img, int y, int x) const { return (size_t)((int64_t)img * stride + (int64_t)y * pitch + x); }
};
inline SrcPlane packed_plane(const void* data, int row_elems, int h) { return {data, row_elems, (int64_t)row_elems * h}; }

// pyramid.cu: the remap of n frames through a rectifier and / or a depth registration into packed float32 planes dI / dZ of
// the target's w*h floats per image (the registration's if any, else the rectifier's output).  raw as in
// pyramid_build_batch_input.  Through a rectifier, I (and M) have its input size and go through its map, and with M.data the
// remapped byte masks (1 = usable) go to dM; without one, I and M are the registration's w x h and the build reads M in
// place.  With a registration, Z is the depth camera's dw x dh and dZ its z-buffer first.
int remap_batch(dvo_b200_ctx* ctx, const dvo_b200_rectifier* rect, const dvo_b200_depth_registration* reg, int n, SrcPlane I,
                SrcPlane Z, int raw, float zscale, SrcPlane M, float* dI, float* dZ, uint8_t* dM);
// I / Z: level-0 intensity and depth (raw == 0: float32 / float32 metres; raw == 1: 8-bit grey / 16-bit raw depth).  M: the
// masks (bytes, nonzero = usable), or M.data == NULL for none; mask_roles: DVO_B200_MASK_ROLE_* bits (ignored without masks).
// K: level 0's fx, fy, ox, oy.  The selection has the default thresholds.  The build reads I, Z and M in place until its
// last kernel has run.
int pyramid_build_batch_input(dvo_b200_ctx* ctx, int n, SrcPlane I, SrcPlane Z, int raw, float zscale, int w, int h,
                              const float K[4], int levels, dvo_b200_pyramid** out, SrcPlane M, int mask_roles);
int pyramid_reselect(dvo_b200_ctx* ctx, dvo_b200_pyramid* p, float ti, float td);
void wait_for_pyramid(dvo_b200_ctx* ctx, const dvo_b200_pyramid* p);   // order ctx's stream after the pyramid's build / re-selection
int note_foreign_use(dvo_b200_ctx* ctx, const dvo_b200_pyramid* p);    // after enqueueing work that reads p (see Slab::foreign_uses)
void pyramid_free(dvo_b200_pyramid* p);
void pool_close(dvo_b200_ctx* ctx);
int ensure_stage(dvo_b200_ctx* ctx, size_t dev_bytes, size_t host_bytes);

// tracker.cu.  The two calls below run the level kernel in legs (tracker.cu: Leg), each one run over a range of pyramid
// levels of a batch of pairs, through one path: check_batch and begin_call, ensure_workspace, stage_inputs, launch_segments,
// end_call.  A match is one leg, a multi-hypothesis match two, and a test hook one leg of one pair at one level.
// One match of n pairs (refs[i], curs[i]) after its entry point's argument checks (capi.cu).  k = 0: a plain match; k >= 1:
// dvo_b200_match_batch_hypotheses[_modes] (checked by hypotheses_args.h), whose per-pair inputs are per hypothesis, n * k.
// A field left at its default is an input the call does not have or an output it does not want.
struct MatchCall {
  const dvo_b200_config* cfg = nullptr;  // levels, iterations, thresholds of every alignment of the call
  int n = 0;                             // pairs
  dvo_b200_pyramid* const* refs = nullptr;   // the reference pyramid of each pair
  dvo_b200_pyramid* const* curs = nullptr;   // the current pyramid of each pair
  const double* T_init = nullptr;        // row-major 4 x 4 initial estimates (host): n, or with k >= 1 the n * k hypotheses
  int k = 0;                             // hypotheses per pair, screened on levels first .. screen_level; 0: a plain match
  int screen_level = 0;                  // k >= 1: the last level of the screening
  double min_ratio = 0.0;                // k >= 1: hypothesis_score's minimum ratio of constraints to valid pixels
  const double* prior = nullptr;         // a motion prior: row-major 6 x 6 informations (host) in place of cfg->mu I (then 0)
  const double* ab_init = nullptr;       // photometric mode: the starting (alpha, beta) (host, 2 doubles each), NULL = (1, 0)
  dvo_b200_result* results = nullptr;    // n
  double* ab_out = nullptr;              // != NULL: the photometric mode (pose, gain, bias); final (alpha, beta) (2n)
  double* screen_ab = nullptr;           // k >= 1, photometric: (alpha, beta) where each screening run ended (2nk)
  int32_t* best = nullptr;               // k >= 1: the chosen hypothesis of each pair (n)
  double* scores = nullptr;              // k >= 1: the score of each hypothesis (nk)
  dvo_b200_result* screen_results = nullptr;   // k >= 1: the result of each screening run (nk)
  dvo_b200_iteration_stats* iter_stats = nullptr;   // iteration logs (max_log per pair)
  int max_log = 0;                       // entries per pair of iter_stats (ignored without it)
  const dvo_b200_weight_maps* maps = nullptr;   // also the weight maps (weight_maps.cu) of the returned alignments
  // false: every output above is host memory, and the call returns once they hold the results.  true: every output is
  // device memory of the context's device (maps: DVO_B200_MAPS_DEVICE); the call enqueues its work and returns, and its
  // level flags surface at dvo_b200_synchronize.
  bool device_outputs = false;
};
int tracker_match(dvo_b200_ctx* ctx, const MatchCall& c);
PyramidView pyramid_view(const dvo_b200_pyramid* p, int level);   // what modes_args.h reads of a pyramid
int check_level_flags(dvo_b200_ctx* ctx);   // after a stream synchronisation: did a level kernel report a timeout?
// The test hooks: one iteration at T (staged as the leg's initial estimate and placed into the state by k_set_state).
int tracker_linearize(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* ref, dvo_b200_pyramid* cur,
                      int level, const double* T, int use_weights, const float* prev_precision, int64_t* count,
                      float* precision_out, float* ll_out, double* A_out, double* b_out, float* planes7,
                      const double* ab = nullptr);   // ab != NULL: photometric mode at (alpha, beta); A_out 8 x 8, b_out 8

// weight_maps.cu, the weight maps of a match (maps checked by maps_args.h).  prepare: before the match's first launch, the
// device scratch of DVO_B200_MAPS_HOST.  launch: k_weight_maps on the batch's final pair states d_states, after the level kernels
// and k_finalize (level = cfg->last_level; d_pls: the batch's descriptors of that level; d_affine: the photometric mode's
// brightness states, or NULL; all three in the pair slots of the leg the results come from); a launch error surfaces at the caller's next cudaGetLastError.  copy_back: with
// DVO_B200_MAPS_HOST, the copies into the caller's host layout, before the call's synchronisation.
int weight_maps_prepare(dvo_b200_ctx* ctx, const dvo_b200_weight_maps& maps, int n, const dvo_b200_pyramid* ref0, int level);
void weight_maps_launch(dvo_b200_ctx* ctx, const dvo_b200_weight_maps& maps, int n, const dvo_b200_pyramid* ref0, int level,
                        const PairState* d_states, const PairLevel* d_pls, const AffineState* d_affine);
int weight_maps_copy_back(dvo_b200_ctx* ctx, const dvo_b200_weight_maps& maps, int n, const dvo_b200_pyramid* ref0, int level);

}  // namespace dvo_b200
