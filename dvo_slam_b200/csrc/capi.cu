// capi.cu -- the extern "C" surface declared in include/dvo_b200.h.
#include "common.cuh"
#include "hypotheses_args.h"
#include "maps_args.h"
#include "prior_args.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <vector>

namespace dvo_b200 {

int set_error(dvo_b200_ctx* ctx, int code, const std::string& msg) {
  if (ctx) ctx->last_error = msg;
  return code;
}

int check_cuda(dvo_b200_ctx* ctx, cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  std::string msg = std::string("CUDA error: ") + cudaGetErrorString(e) + " in " + what;
  cudaGetLastError();
  return set_error(ctx, e == cudaErrorMemoryAllocation ? DVO_B200_ERR_OUT_OF_MEMORY : DVO_B200_ERR_CUDA, msg);
}

static cudaEvent_t get_event(dvo_b200_ctx* ctx) {
  if (!ctx->event_pool.empty()) { cudaEvent_t e = ctx->event_pool.back(); ctx->event_pool.pop_back(); return e; }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

ProfScope::ProfScope(dvo_b200_ctx* c, int cls_, int nlaunch) : ctx(c), cls(cls_) {
  if (!ctx->profile) return;
  a = get_event(ctx); b = get_event(ctx);
  cudaEventRecord(a, ctx->stream);
  ctx->prof_launches[cls] += nlaunch;
}
ProfScope::~ProfScope() {
  if (!a) return;
  cudaEventRecord(b, ctx->stream);
  ctx->prof_pending.push_back({cls, {a, b}});
}

static void drain_profile(dvo_b200_ctx* ctx) {
  for (auto& e : ctx->prof_pending) {
    float ms = 0.f;
    cudaEventSynchronize(e.second.second);
    cudaEventElapsedTime(&ms, e.second.first, e.second.second);
    ctx->prof_ms[e.first] += ms;
    ctx->event_pool.push_back(e.second.first);
    ctx->event_pool.push_back(e.second.second);
  }
  ctx->prof_pending.clear();
}

namespace {

__global__ void k_convert_bgr(SrcPlane bgr, uint8_t* __restrict__ grey, int w, int h) {
  // benchmark_slam.cpp:58-68: cv::cvtColor(rgb, grey, CV_BGR2GRAY) on CV_8UC3 (convertTo(CV_32F) happens in the pyramid
  // kernels' loads).  OpenCV's 8-bit path is fixed point: (B*1868 + G*9617 + R*4899 + (1 << 13)) >> 14.
  // bgr: interleaved, 3 elements per pixel; grey: packed, image img at img * w * h.
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w * h) return;
  const int y = i / w, x = i - y * w;
  const uint8_t* p = reinterpret_cast<const uint8_t*>(bgr.data) + bgr.at(img, y, 3 * x);
  grey[(size_t)img * w * h + i] = (uint8_t)((1868 * (int)p[0] + 9617 * (int)p[1] + 4899 * (int)p[2] + 8192) >> 14);
}

// n BGR images -> n packed 8-bit grey images, as cv::cvtColor leaves them.  The level-0 kernels then read the grey plane (each
// grey pixel several times: the 2x2 mean and the five taps of the central differences).
void convert_bgr(dvo_b200_ctx* ctx, int n, int w, int h, SrcPlane bgr, uint8_t* grey) {
  k_convert_bgr<<<dim3((unsigned)(((size_t)w * h + 255) / 256), n), 256, 0, ctx->stream>>>(bgr, grey, w, h);
  ctx->launches++;
}

}  // namespace

// One dvo_b200_device_plane of n images of width x height pixels, elem bytes per element and per_px elements per pixel ->
// the SrcPlane the pyramid kernels read.  Every check of the header's list; the pointer checks look at the first and the
// last byte of the plane's extent.
static int device_plane(dvo_b200_ctx* ctx, const char* fn, const dvo_b200_device_plane* p, const char* name, int elem, int per_px,
                        int n, int width, int height, SrcPlane* out) {
  auto bad = [&](const std::string& why) {
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, std::string(fn) + ": " + name + ": " + why);
  };
  if (!p || !p->data) return bad("null plane or data pointer");
  const int64_t row = (int64_t)width * per_px * elem;
  if (p->row_bytes < row)
    return bad("row_bytes " + std::to_string(p->row_bytes) + " < width * bytes per pixel = " + std::to_string(row));
  if (p->row_bytes % elem) return bad("row_bytes " + std::to_string(p->row_bytes) + " is not a multiple of " + std::to_string(elem));
  if (p->image_bytes < 0) return bad("negative image_bytes " + std::to_string(p->image_bytes));
  if (p->image_bytes % elem)
    return bad("image_bytes " + std::to_string(p->image_bytes) + " is not a multiple of " + std::to_string(elem));
  if ((uintptr_t)p->data % elem) return bad("data is not aligned to its " + std::to_string(elem) + "-byte elements");
  int64_t a = 0, b = 0, last = 0;
  if (__builtin_mul_overflow((int64_t)(n - 1), p->image_bytes, &a) || __builtin_mul_overflow((int64_t)(height - 1), p->row_bytes, &b) ||
      __builtin_add_overflow(a, b, &last) || __builtin_add_overflow(last, row - 1, &last) ||
      (uintptr_t)p->data + (uint64_t)last < (uintptr_t)p->data)
    return bad("the extent of the plane overflows");
  const char* ends[2] = {(const char*)p->data, (const char*)p->data + last};
  for (const char* q : ends) {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, q) != cudaSuccess) { cudaGetLastError(); return bad("not a CUDA pointer"); }
    if (attr.type != cudaMemoryTypeDevice && attr.type != cudaMemoryTypeManaged)
      return bad(attr.type == cudaMemoryTypeHost ? "pinned host memory, not device memory" : "host memory, not device memory");
    if (attr.device != ctx->device)
      return bad("memory of device " + std::to_string(attr.device) + ", the context is on device " + std::to_string(ctx->device));
  }
  *out = SrcPlane{p->data, p->row_bytes / elem, p->image_bytes / elem};
  return 0;
}


// The context's staging memory for one create, in 256-byte aligned sections: the uploaded frames (depth, then the image, then
// 64 bytes of slack), the uploaded masks, the grey reduced from BGR, then the remapped or registered planes (float32
// intensity and depth of level 0 and, through a rectifier, its byte masks).  A section the call does not need has size 0;
// a device create uploads nothing.
struct StageLayout {
  size_t image, masks, grey, remap, total;   // byte offsets (the depth frames start at 0) and the bytes of all sections
};

static StageLayout stage_layout(const CreateArgs& a, int w0, int h0) {
  auto up = [](size_t v) { return (v + 255) / 256 * 256; };
  const bool f32 = a.format == DVO_B200_INPUT_FLOAT32, bgr = a.format == DVO_B200_INPUT_BGR8_DEPTH16;
  const bool masked = a.device ? a.mask_plane != nullptr : a.masks != nullptr;
  const size_t npx = (size_t)a.width * a.height * a.n;
  const size_t dnpx = a.reg ? (size_t)a.reg->dw * a.reg->dh * a.n : npx;
  StageLayout s{};
  size_t end = 0;
  if (!a.device) {
    s.image = up(dnpx * (f32 ? 4 : 2));
    end = s.image + npx * (f32 ? 4 : bgr ? 3 : 1) + 64;
    s.masks = up(end);
    if (masked) end = s.masks + npx;
  }
  s.grey = up(end);
  if (bgr) end = s.grey + npx;
  s.remap = up(end);
  if (a.rect || a.reg) end = s.remap + (size_t)w0 * h0 * a.n * (2 * sizeof(float) + (a.rect && masked ? 1 : 0));
  s.total = end;
  return s;
}

// Every create: the checks of create_args.h and the device planes' before any device work, then the upload into staging
// (host forms), the BGR reduction, the remap or registration, and the build.  The frames stay in their file representation:
// the pyramid kernels convert in their loads (no float32 copy of a raw frame is written); BGR is reduced to 8-bit grey
// first, as cv::cvtColor leaves it.  Device planes are read in place.
static int create_pyramids(dvo_b200_ctx* ctx, const CreateArgs& a, dvo_b200_pyramid** out) {
  const std::string why = create_args_error(ctx, a, out);
  if (!why.empty()) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, why);
  cudaSetDevice(ctx->device);
  const bool f32 = a.format == DVO_B200_INPUT_FLOAT32, bgr = a.format == DVO_B200_INPUT_BGR8_DEPTH16;
  const int n = a.n, w = a.width, h = a.height;
  const int dw = a.reg ? a.reg->dw : w, dh = a.reg ? a.reg->dh : h;   // with a registration, depth has the depth camera's size
  SrcPlane I, Z, M{nullptr, 0, 0};
  if (a.device) {
    int rc = device_plane(ctx, a.fn, a.image_plane, "image", f32 ? 4 : 1, bgr ? 3 : 1, n, w, h, &I);
    if (!rc) rc = device_plane(ctx, a.fn, a.depth_plane, "depth", f32 ? 4 : 2, 1, n, dw, dh, &Z);
    if (!rc && a.mask_plane) rc = device_plane(ctx, a.fn, a.mask_plane, "masks", 1, 1, n, w, h, &M);
    if (rc) return rc;
  }
  int w0, h0;
  const float* K;
  create_level0(a, &w0, &h0, &K);
  const StageLayout s = stage_layout(a, w0, h0);
  if (int rc = ensure_stage(ctx, s.total, 0)) return rc;
  char* stage = (char*)ctx->d_stage;
  if (!a.device) {
    const size_t npx = (size_t)w * h * n;
    const size_t zbytes = (size_t)dw * dh * n * (f32 ? 4 : 2), ibytes = npx * (f32 ? 4 : bgr ? 3 : 1);
    DVO_CUDA(ctx, cudaMemcpyAsync(stage, a.depth, zbytes, cudaMemcpyHostToDevice, ctx->stream));
    DVO_CUDA(ctx, cudaMemcpyAsync(stage + s.image, a.image, ibytes, cudaMemcpyHostToDevice, ctx->stream));
    ctx->h2d_bytes += zbytes + ibytes;
    Z = packed_plane(stage, dw, dh);
    I = packed_plane(stage + s.image, bgr ? 3 * w : w, h);
    if (a.masks) {
      DVO_CUDA(ctx, cudaMemcpyAsync(stage + s.masks, a.masks, npx, cudaMemcpyHostToDevice, ctx->stream));
      ctx->h2d_bytes += npx;
      M = packed_plane(stage + s.masks, w, h);
    }
  }
  if (bgr) {
    convert_bgr(ctx, n, w, h, I, (uint8_t*)stage + s.grey);
    I = packed_plane(stage + s.grey, w, h);
  }
  int raw = f32 ? 0 : 1;
  float zscale = f32 ? 0.f : a.depth_scale;
  if (a.rect || a.reg) {   // the build reads the packed float32 planes of level 0 (and the remapped masks through a rectifier)
    const size_t npx0 = (size_t)w0 * h0 * n;
    float* dI = (float*)(stage + s.remap);
    float* dZ = dI + npx0;
    uint8_t* dM = a.rect && M.data ? (uint8_t*)(dZ + npx0) : nullptr;
    if (int rc = remap_batch(ctx, a.rect, a.reg, n, I, Z, raw, zscale, M, dI, dZ, dM)) return rc;
    I = packed_plane(dI, w0, h0);
    Z = packed_plane(dZ, w0, h0);
    raw = 0;
    zscale = 0.f;
    if (a.rect) M = dM ? packed_plane(dM, w0, h0) : SrcPlane{nullptr, 0, 0};
  }
  return pyramid_build_batch_input(ctx, n, I, Z, raw, zscale, w0, h0, K, a.levels, out, M, a.roles);
}

static CreateArgs host_args(const char* fn, int n, int format, const void* image, const void* depth, float depth_scale,
                            const uint8_t* masks, int roles, int width, int height, int levels) {
  CreateArgs a;
  a.fn = fn; a.n = n; a.format = format; a.image = image; a.depth = depth; a.depth_scale = depth_scale; a.masks = masks;
  a.roles = roles; a.width = width; a.height = height; a.levels = levels;
  return a;
}

static CreateArgs device_args(const char* fn, int n, int format, const dvo_b200_device_plane* image, const dvo_b200_device_plane* depth,
                              float depth_scale, const dvo_b200_device_plane* masks, int roles, int width, int height, int levels) {
  CreateArgs a = host_args(fn, n, format, nullptr, nullptr, depth_scale, nullptr, roles, width, height, levels);
  a.device = true; a.image_plane = image; a.depth_plane = depth; a.mask_plane = masks;
  return a;
}

static CreateArgs with_K(CreateArgs a, float fx, float fy, float ox, float oy) {
  a.K[0] = fx; a.K[1] = fy; a.K[2] = ox; a.K[3] = oy;
  return a;
}

static CreateArgs with_remap(CreateArgs a, int remap, const dvo_b200_rectifier* rect, const dvo_b200_depth_registration* reg) {
  a.remap = remap;
  a.rect = rect; a.reg = reg;
  return a;
}

}  // namespace dvo_b200

using namespace dvo_b200;

extern "C" {

int dvo_b200_abi_version(void) { return DVO_B200_ABI_VERSION; }

int dvo_b200_create(int device, void* stream, dvo_b200_ctx** out) {
  if (!out) return DVO_B200_ERR_INVALID_ARGUMENT;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) {
    cudaGetLastError();
    return DVO_B200_ERR_CUDA;   // no CPU fallback: without a CUDA device there is no engine
  }
  if (cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return DVO_B200_ERR_CUDA; }
  static std::atomic<uint64_t> next_uid{1};
  dvo_b200_ctx* ctx = new dvo_b200_ctx;
  ctx->device = device;
  ctx->uid = next_uid.fetch_add(1, std::memory_order_relaxed);
  ctx->pool = std::make_shared<SlabPool>();
  ctx->pool->device = device;
  if (stream) { ctx->stream = (cudaStream_t)stream; ctx->own_stream = false; }
  else {
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); delete ctx; return DVO_B200_ERR_CUDA; }
    ctx->own_stream = true;
  }
  if (getenv("DVO_B200_TIMING")) {
    cudaMalloc((void**)&ctx->d_dbg, sizeof(unsigned long long) * 256);
    cudaMemset(ctx->d_dbg, 0, sizeof(unsigned long long) * 256);
    for (int l = 0; l < 8; ++l) { unsigned long long big = ~0ull; cudaMemcpy(ctx->d_dbg + 128 + 8 * l + 6, &big, 8, cudaMemcpyHostToDevice); }
  }
  *out = ctx;
  return 0;
}

int dvo_b200_destroy(dvo_b200_ctx* ctx) {
  if (!ctx) return DVO_B200_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  cudaStreamSynchronize(ctx->stream);
  drain_profile(ctx);
  for (cudaEvent_t e : ctx->event_pool) cudaEventDestroy(e);
  Workspace& ws = ctx->ws;
  cudaFree(ws.d_pair_level); cudaFree(ws.d_state); cudaFree(ws.d_scratch); cudaFree(ws.d_dump); cudaFree(ws.d_tinit);
  cudaFree(ws.d_iter_log); cudaFree(ws.d_csat); cudaFree(ws.d_prior); cudaFree(ws.d_maps);
  if (ws.h_active) cudaFreeHost(ws.h_active);
  pool_close(ctx);
  cudaFree(ctx->d_stage);
  if (ctx->h_stage) cudaFreeHost(ctx->h_stage);
  if (ctx->h_results) cudaFreeHost(ctx->h_results);
  if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
  cudaGetLastError();
  delete ctx;
  return 0;
}

void* dvo_b200_stream(dvo_b200_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

int dvo_b200_synchronize(dvo_b200_ctx* ctx) {
  if (!ctx) return DVO_B200_ERR_INVALID_ARGUMENT;
  DVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return check_level_flags(ctx);   // a timeout inside dvo_b200_match_batch_device surfaces here
}

const char* dvo_b200_last_error(dvo_b200_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }

void dvo_b200_config_default(dvo_b200_config* cfg) {
  if (!cfg) return;
  // dense_tracking_config.cpp:27-42
  cfg->first_level = 3; cfg->last_level = 1; cfg->max_iterations_per_level = 100; cfg->use_initial_estimate = 0;
  cfg->precision = 5e-7; cfg->mu = 0.0; cfg->intensity_derivative_threshold = 0.0f; cfg->depth_derivative_threshold = 0.0f;
}

int64_t dvo_b200_kernel_launches(dvo_b200_ctx* ctx) { return ctx ? ctx->launches : 0; }
int64_t dvo_b200_h2d_bytes(dvo_b200_ctx* ctx) { return ctx ? ctx->h2d_bytes : 0; }
int64_t dvo_b200_d2h_bytes(dvo_b200_ctx* ctx) { return ctx ? ctx->d2h_bytes : 0; }

int dvo_b200_set_estimator(dvo_b200_ctx* ctx, int32_t estimator) {
  if (!ctx) return DVO_B200_ERR_INVALID_ARGUMENT;
  if (estimator != DVO_B200_ESTIMATOR_REFERENCE && estimator != DVO_B200_ESTIMATOR_CORRECTED)
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "set_estimator: unknown estimator " + std::to_string(estimator));
  ctx->estimator = estimator;
  return 0;
}

int dvo_b200_get_estimator(const dvo_b200_ctx* ctx) { return ctx ? ctx->estimator : DVO_B200_ERR_INVALID_ARGUMENT; }

int dvo_b200_pyramid_create_batch(dvo_b200_ctx* ctx, int32_t n, const float* intensity, const float* depth, int32_t width,
                                  int32_t height, float fx, float fy, float ox, float oy, int32_t levels,
                                  dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_K(host_args("pyramid_create", n, DVO_B200_INPUT_FLOAT32, intensity, depth, 0.f, nullptr,
                                               DVO_B200_MASK_ROLE_REFERENCE, width, height, levels), fx, fy, ox, oy), out);
}

int dvo_b200_pyramid_create(dvo_b200_ctx* ctx, const float* intensity, const float* depth, int32_t width, int32_t height,
                            float fx, float fy, float ox, float oy, int32_t levels, dvo_b200_pyramid** out) {
  return dvo_b200_pyramid_create_batch(ctx, 1, intensity, depth, width, height, fx, fy, ox, oy, levels, out);
}

int dvo_b200_pyramid_create_raw_batch(dvo_b200_ctx* ctx, int32_t n, const uint8_t* grey, const uint16_t* raw_depth,
                                      float depth_scale, int32_t width, int32_t height, float fx, float fy, float ox,
                                      float oy, int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_K(host_args("pyramid_create_raw", n, DVO_B200_INPUT_GREY8_DEPTH16, grey, raw_depth, depth_scale,
                                               nullptr, DVO_B200_MASK_ROLE_REFERENCE, width, height, levels), fx, fy, ox, oy), out);
}

int dvo_b200_pyramid_create_bgr_batch(dvo_b200_ctx* ctx, int32_t n, const uint8_t* bgr, const uint16_t* raw_depth,
                                      float depth_scale, int32_t width, int32_t height, float fx, float fy, float ox,
                                      float oy, int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_K(host_args("pyramid_create_bgr", n, DVO_B200_INPUT_BGR8_DEPTH16, bgr, raw_depth, depth_scale,
                                               nullptr, DVO_B200_MASK_ROLE_REFERENCE, width, height, levels), fx, fy, ox, oy), out);
}

int dvo_b200_pyramid_create_masked_batch(dvo_b200_ctx* ctx, int32_t n, int32_t format, const void* image, const void* depth,
                                         float depth_scale, const uint8_t* masks, int32_t width, int32_t height, float fx,
                                         float fy, float ox, float oy, int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_K(host_args("pyramid_create_masked", n, format, image, depth, depth_scale, masks,
                                               DVO_B200_MASK_ROLE_REFERENCE, width, height, levels), fx, fy, ox, oy), out);
}

int dvo_b200_pyramid_create_masked_batch_roles(dvo_b200_ctx* ctx, int32_t n, int32_t format, const void* image,
                                               const void* depth, float depth_scale, const uint8_t* masks, int32_t roles,
                                               int32_t width, int32_t height, float fx, float fy, float ox, float oy,
                                               int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_K(host_args("pyramid_create_masked_roles", n, format, image, depth, depth_scale, masks, roles,
                                               width, height, levels), fx, fy, ox, oy), out);
}

int dvo_b200_pyramid_create_device_batch(dvo_b200_ctx* ctx, int32_t n, int32_t format, const dvo_b200_device_plane* image,
                                         const dvo_b200_device_plane* depth, float depth_scale, const dvo_b200_device_plane* masks,
                                         int32_t roles, int32_t width, int32_t height, float fx, float fy, float ox, float oy,
                                         int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_K(device_args("pyramid_create_device", n, format, image, depth, depth_scale, masks, roles, width,
                                                 height, levels), fx, fy, ox, oy), out);
}

int dvo_b200_undistort_map(int32_t width, int32_t height, const double K[4], const double dist[5], const double K_new[4],
                           float* map_x, float* map_y) {
  if (width <= 0 || height <= 0 || !K || !dist || !K_new || !map_x || !map_y) return DVO_B200_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < 5; ++i)
    if (!std::isfinite(dist[i]) || (i < 4 && (!std::isfinite(K[i]) || !std::isfinite(K_new[i])))) return DVO_B200_ERR_INVALID_ARGUMENT;
  const double fx = K[0], fy = K[1], cx = K[2], cy = K[3], nfx = K_new[0], nfy = K_new[1], ncx = K_new[2], ncy = K_new[3];
  const double k1 = dist[0], k2 = dist[1], p1 = dist[2], p2 = dist[3], k3 = dist[4];
  const double sx = fx / nfx, sy = fy / nfy;
  for (int v = 0; v < height; ++v) {
    const double y = (v - ncy) / nfy;
    for (int u = 0; u < width; ++u) {
      // the order of the header comment, term by term
      const double x = (u - ncx) / nfx;
      const double r2 = x * x + y * y;
      const double kr = ((k3 * r2 + k2) * r2 + k1) * r2;
      const double dx = x * kr + ((2 * p1) * x * y + p2 * (r2 + 2 * x * x));
      const double dy = y * kr + (p1 * (r2 + 2 * y * y) + (2 * p2) * x * y);
      map_x[(size_t)v * width + u] = (float)((cx + sx * (u - ncx)) + fx * dx);
      map_y[(size_t)v * width + u] = (float)((cy + sy * (v - ncy)) + fy * dy);
    }
  }
  return 0;
}

int dvo_b200_rectifier_create(dvo_b200_ctx* ctx, int32_t in_width, int32_t in_height, int32_t width, int32_t height,
                              const float* map_x, const float* map_y, const float K_new[4], dvo_b200_rectifier** out) {
  if (out) *out = nullptr;
  if (!ctx || !map_x || !map_y || !K_new || !out || in_width < 2 || in_height < 2 || width <= 0 || height <= 0)
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "rectifier_create: null/invalid argument");
  cudaSetDevice(ctx->device);
  const size_t npx = (size_t)width * height;
  float* d = nullptr;
  DVO_CUDA(ctx, cudaMallocAsync((void**)&d, 2 * npx * sizeof(float), ctx->stream));
  cudaError_t e = cudaMemcpyAsync(d, map_x, npx * sizeof(float), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d + npx, map_y, npx * sizeof(float), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);   // the caller's arrays may go when this returns
  if (e != cudaSuccess) {
    cudaFreeAsync(d, ctx->stream);
    return check_cuda(ctx, e, "rectifier_create: map upload");
  }
  ctx->h2d_bytes += 2 * npx * sizeof(float);
  dvo_b200_rectifier* r = new dvo_b200_rectifier;
  r->ctx = ctx; r->in_w = in_width; r->in_h = in_height; r->w = width; r->h = height; r->map = d;
  for (int i = 0; i < 4; ++i) r->K[i] = K_new[i];
  *out = r;
  return 0;
}

int dvo_b200_rectifier_release(dvo_b200_rectifier* r) {
  if (!r) return DVO_B200_ERR_INVALID_ARGUMENT;
  DeviceScope dev(r->ctx->device);
  // every create that read the map was enqueued on this stream before this call: the free follows them in stream order
  const cudaError_t e = cudaFreeAsync(r->map, r->ctx->stream);
  const int rc = check_cuda(r->ctx, e, "rectifier_release");
  delete r;
  return rc;
}

int dvo_b200_pyramid_create_rectified_batch(dvo_b200_ctx* ctx, const dvo_b200_rectifier* rect, int32_t n, int32_t format,
                                            const void* image, const void* depth, float depth_scale, const uint8_t* masks,
                                            int32_t roles, int32_t width, int32_t height, int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_remap(host_args("pyramid_create_rectified", n, format, image, depth, depth_scale, masks, roles,
                                                   width, height, levels), kRemapRectify, rect, nullptr), out);
}

int dvo_b200_pyramid_create_rectified_device_batch(dvo_b200_ctx* ctx, const dvo_b200_rectifier* rect, int32_t n, int32_t format,
                                                   const dvo_b200_device_plane* image, const dvo_b200_device_plane* depth,
                                                   float depth_scale, const dvo_b200_device_plane* masks, int32_t roles, int32_t width,
                                                   int32_t height, int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_remap(device_args("pyramid_create_rectified_device", n, format, image, depth, depth_scale, masks,
                                                     roles, width, height, levels), kRemapRectify, rect, nullptr), out);
}

int dvo_b200_depth_rays(int32_t dw, int32_t dh, const double K[4], const double dist[5], float* cx_ray, float* cy_ray, float* kx_ray,
                        float* ky_ray) {
  if (dw < 2 || dh < 2 || !K || !cx_ray || !cy_ray || !kx_ray || !ky_ray) return DVO_B200_ERR_INVALID_ARGUMENT;
  for (int i = 0; i < 5; ++i)
    if ((i < 4 && !std::isfinite(K[i])) || (dist && !std::isfinite(dist[i]))) return DVO_B200_ERR_INVALID_ARGUMENT;
  const double fx = K[0], fy = K[1], cx = K[2], cy = K[3];
  if (!(fx > 0) || !(fy > 0)) return DVO_B200_ERR_INVALID_ARGUMENT;
  // the ray through pixel coordinates (u, v): the order of the header comment, term by term
  auto ray = [&](double u, double v, float* rx, float* ry) {
    const double xd = (u - cx) / fx, yd = (v - cy) / fy;
    double x = xd, y = yd;
    if (dist) {
      const double k1 = dist[0], k2 = dist[1], p1 = dist[2], p2 = dist[3], k3 = dist[4];
      for (int it = 0;; ++it) {
        const double r2 = x * x + y * y;
        const double R = 1 + ((k3 * r2 + k2) * r2 + k1) * r2;
        const double dR = k1 + (2 * k2 + 3 * k3 * r2) * r2;
        const double ex = x * R + 2 * p1 * x * y + p2 * (r2 + 2 * x * x) - xd;
        const double ey = y * R + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y - yd;
        if (std::fabs(ex) < 1e-12 && std::fabs(ey) < 1e-12) break;
        if (it == DVO_B200_DEPTH_RAYS_MAX_ITER) return false;
        const double a = R + 2 * x * x * dR + 2 * p1 * y + 6 * p2 * x;
        const double b = 2 * x * y * dR + 2 * p1 * x + 2 * p2 * y;
        const double d = R + 2 * y * y * dR + 6 * p1 * y + 2 * p2 * x;
        const double det = a * d - b * b;
        const double nx = x - (d * ex - b * ey) / det, ny = y - (a * ey - b * ex) / det;
        x = nx;
        y = ny;
      }
    }
    *rx = (float)x;
    *ry = (float)y;
    return true;
  };
  for (int v = 0; v < dh; ++v)
    for (int u = 0; u < dw; ++u)
      if (!ray(u, v, cx_ray + (size_t)v * dw + u, cy_ray + (size_t)v * dw + u)) return DVO_B200_ERR_INVALID_ARGUMENT;
  for (int v = 0; v <= dh; ++v)
    for (int u = 0; u <= dw; ++u)
      if (!ray(u - 0.5, v - 0.5, kx_ray + (size_t)v * (dw + 1) + u, ky_ray + (size_t)v * (dw + 1) + u)) return DVO_B200_ERR_INVALID_ARGUMENT;
  return 0;
}

int dvo_b200_depth_registration_create(dvo_b200_ctx* ctx, int32_t dw, int32_t dh, const float* cx_ray, const float* cy_ray,
                                       const float* kx_ray, const float* ky_ray, const double T[16], int32_t width, int32_t height,
                                       const float K[4], dvo_b200_depth_registration** out) {
  if (out) *out = nullptr;
  auto bad = [&](const char* why) {
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, std::string("depth_registration_create: ") + why);
  };
  if (!ctx || !cx_ray || !cy_ray || !kx_ray || !ky_ray || !T || !K || !out || dw < 2 || dh < 2 || width <= 0 || height <= 0)
    return bad("null/invalid argument");
  for (int i = 0; i < 16; ++i)
    if (!std::isfinite(T[i])) return bad("non-finite T_color_depth");
  if (T[12] != 0 || T[13] != 0 || T[14] != 0 || T[15] != 1) return bad("T_color_depth: bottom row is not (0, 0, 0, 1)");
  double err = 0;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) {
      double s = 0;
      for (int k = 0; k < 3; ++k) s += T[4 * k + a] * T[4 * k + b];
      err = std::max(err, std::fabs(s - (a == b ? 1.0 : 0.0)));
    }
  const double det = T[0] * (T[5] * T[10] - T[6] * T[9]) - T[1] * (T[4] * T[10] - T[6] * T[8]) + T[2] * (T[4] * T[9] - T[5] * T[8]);
  if (!(err <= 1e-6) || !(det > 0)) return bad("T_color_depth is not a rigid transform (R^T R != I or det R <= 0)");
  for (int i = 0; i < 4; ++i)
    if (!std::isfinite(K[i])) return bad("non-finite K");
  if (!(K[0] > 0) || !(K[1] > 0)) return bad("non-positive focal length");
  const size_t nc = (size_t)dw * dh, nk = (size_t)(dw + 1) * (dh + 1);
  const float* tables[4] = {cx_ray, cy_ray, kx_ray, ky_ray};
  for (int t = 0; t < 4; ++t)
    for (size_t i = 0; i < (t < 2 ? nc : nk); ++i)
      if (!std::isfinite(tables[t][i])) return bad("non-finite ray");
  cudaSetDevice(ctx->device);
  const size_t bytes = (2 * nc + 2 * nk) * sizeof(float);
  float* d = nullptr;
  DVO_CUDA(ctx, cudaMallocAsync((void**)&d, bytes, ctx->stream));
  const size_t offs[4] = {0, nc, 2 * nc, 2 * nc + nk};
  cudaError_t e = cudaSuccess;
  for (int t = 0; t < 4 && e == cudaSuccess; ++t)
    e = cudaMemcpyAsync(d + offs[t], tables[t], (t < 2 ? nc : nk) * sizeof(float), cudaMemcpyHostToDevice, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);   // the caller's arrays may go when this returns
  if (e != cudaSuccess) {
    cudaFreeAsync(d, ctx->stream);
    return check_cuda(ctx, e, "depth_registration_create: ray upload");
  }
  ctx->h2d_bytes += bytes;
  dvo_b200_depth_registration* r = new dvo_b200_depth_registration;
  r->ctx = ctx; r->dw = dw; r->dh = dh; r->w = width; r->h = height; r->rays = d;
  for (int a = 0; a < 3; ++a) {
    for (int b = 0; b < 3; ++b) r->R[3 * a + b] = (float)T[4 * a + b];
    r->t[a] = (float)T[4 * a + 3];
  }
  for (int i = 0; i < 4; ++i) r->K[i] = K[i];
  *out = r;
  return 0;
}

int dvo_b200_depth_registration_release(dvo_b200_depth_registration* r) {
  if (!r) return DVO_B200_ERR_INVALID_ARGUMENT;
  DeviceScope dev(r->ctx->device);
  // every create that read the rays was enqueued on this stream before this call: the free follows them in stream order
  const cudaError_t e = cudaFreeAsync(r->rays, r->ctx->stream);
  const int rc = check_cuda(r->ctx, e, "depth_registration_release");
  delete r;
  return rc;
}

int dvo_b200_pyramid_create_registered_batch(dvo_b200_ctx* ctx, const dvo_b200_depth_registration* reg, const dvo_b200_rectifier* rect,
                                             int32_t n, int32_t format, const void* image, const void* depth, float depth_scale,
                                             const uint8_t* masks, int32_t roles, int32_t width, int32_t height, int32_t levels,
                                             dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_remap(host_args("pyramid_create_registered", n, format, image, depth, depth_scale, masks, roles,
                                                   width, height, levels), kRemapRegister, rect, reg), out);
}

int dvo_b200_pyramid_create_registered_device_batch(dvo_b200_ctx* ctx, const dvo_b200_depth_registration* reg,
                                                    const dvo_b200_rectifier* rect, int32_t n, int32_t format,
                                                    const dvo_b200_device_plane* image, const dvo_b200_device_plane* depth,
                                                    float depth_scale, const dvo_b200_device_plane* masks, int32_t roles, int32_t width,
                                                    int32_t height, int32_t levels, dvo_b200_pyramid** out) {
  return create_pyramids(ctx, with_remap(device_args("pyramid_create_registered_device", n, format, image, depth, depth_scale, masks,
                                                     roles, width, height, levels), kRemapRegister, rect, reg), out);
}

int dvo_b200_pyramid_mask_roles(const dvo_b200_pyramid* p) { return p ? p->mask_roles : DVO_B200_ERR_INVALID_ARGUMENT; }

int dvo_b200_pyramid_create_raw(dvo_b200_ctx* ctx, const uint8_t* grey, const uint16_t* raw_depth, float depth_scale,
                                int32_t width, int32_t height, float fx, float fy, float ox, float oy, int32_t levels,
                                dvo_b200_pyramid** out) {
  return dvo_b200_pyramid_create_raw_batch(ctx, 1, grey, raw_depth, depth_scale, width, height, fx, fy, ox, oy, levels, out);
}

int dvo_b200_pyramid_device(const dvo_b200_pyramid* p) { return p ? p->device : -1; }

int dvo_b200_pyramid_retain(dvo_b200_pyramid* p) {
  if (!p) return DVO_B200_ERR_INVALID_ARGUMENT;
  p->refcount.fetch_add(1, std::memory_order_relaxed);
  return 0;
}

int dvo_b200_pyramid_release(dvo_b200_pyramid* p) {
  if (!p) return DVO_B200_ERR_INVALID_ARGUMENT;
  if (p->refcount.fetch_sub(1, std::memory_order_acq_rel) == 1) {
    // No synchronisation: the pyramid may be released as soon as the calls that used it have returned, on any context,
    // with their work still queued (dvo_b200_match_batch_device returns before its kernels run).  The slab returns to
    // the owning ctx's pool and is only rewritten by a later build on that ctx's stream, which is ordered after the
    // owner's own queued readers by the stream and after other contexts' queued readers by the events those calls
    // left on the slab (Slab::foreign_uses).  If the owner is gone, the slab is freed once those events complete.
    pyramid_free(p);
  }
  return 0;
}

int dvo_b200_pyramid_num_levels(const dvo_b200_pyramid* p) { return p ? p->levels : DVO_B200_ERR_INVALID_ARGUMENT; }

int dvo_b200_pyramid_level_info(const dvo_b200_pyramid* p, int32_t level, int32_t* width, int32_t* height, float K[4]) {
  if (!p || level < 0 || level >= p->levels) return DVO_B200_ERR_INVALID_ARGUMENT;
  const LevelInfo& L = p->L[level];
  if (width) *width = L.w;
  if (height) *height = L.h;
  if (K) { K[0] = L.fx; K[1] = L.fy; K[2] = L.ox; K[3] = L.oy; }
  return 0;
}

int dvo_b200_pyramid_download(dvo_b200_ctx* ctx, const dvo_b200_pyramid* p, int32_t level, float* planes6) {
  if (!p || !planes6 || level < 0 || level >= p->levels)
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "pyramid_download: invalid argument");
  DeviceScope dev(ctx ? ctx->device : p->device);   // the caller's current device is left as it was
  const LevelInfo& L = p->L[level];
  size_t N = L.n;
  const size_t plane = (size_t)L.pitch * L.h;      // float2 elements per plane, rows padded to the pitch
  const size_t nrec = (size_t)L.nbands * L.nstrips * dvo_b200::kRecF2;
  std::vector<float> tmp(4 * plane), rec(2 * nrec);
  if (ctx) DVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (p->slab && p->slab->ready) DVO_CUDA(ctx, cudaEventSynchronize(p->slab->ready));   // the pyramid's own build has finished
  DVO_CUDA(ctx, cudaMemcpy(tmp.data(), p->planes + L.plane_off, sizeof(float) * 4 * plane, cudaMemcpyDeviceToHost));
  DVO_CUDA(ctx, cudaMemcpy(rec.data(), p->planes + L.rec_off, sizeof(float) * 2 * nrec, cudaMemcpyDeviceToHost));
  if (ctx) ctx->d2h_bytes += sizeof(float) * (4 * plane + 2 * nrec);
  // device layout: P0 = (I, Z'), P2 = (I, Z) row-major; (Ix, Iy) in the reference tile records.  The depth gradients are not
  // stored (the tracker forms them from P2 on the fly): restate calculateDerivativeX/Y<float> on the true depth
  // (rgbd_image.cpp:419-472).
  auto Zt = [&](int y, int x) { return tmp[2 * plane + 2 * ((size_t)y * L.pitch + x) + 1]; };
  for (int y = 0; y < L.h; ++y)
    for (int x = 0; x < L.w; ++x) {
      const size_t o = 2 * ((size_t)y * L.pitch + x), i = (size_t)y * L.w + x;
      const size_t g = 2 * (dvo_b200::rec_cell(x, y, L.nbands) + dvo_b200::kRecP1);
      planes6[0 * N + i] = tmp[o]; planes6[1 * N + i] = tmp[o + 1];
      planes6[2 * N + i] = rec[g]; planes6[3 * N + i] = rec[g + 1];
      const int xp = x > 0 ? x - 1 : 0, xn = x < L.w - 1 ? x + 1 : L.w - 1, yp = y > 0 ? y - 1 : 0, yn = y < L.h - 1 ? y + 1 : L.h - 1;
      const float dzx = Zt(y, xn) - Zt(y, xp), dzy = Zt(yn, x) - Zt(yp, x);
      planes6[4 * N + i] = dzx * 0.5f; planes6[5 * N + i] = dzy * 0.5f;
    }
  return 0;
}

int dvo_b200_pyramid_select(dvo_b200_ctx* ctx, dvo_b200_pyramid* p, int32_t level, float intensity_threshold,
                            float depth_threshold, int64_t* count, uint8_t* mask) {
  if (!ctx || !p || level < 0 || level >= p->levels)
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "pyramid_select: invalid argument");
  cudaSetDevice(ctx->device);
  wait_for_pyramid(ctx, p);   // the build may still be running, on another context's stream
  int rc = pyramid_reselect(ctx, p, intensity_threshold, depth_threshold);
  if (rc) return rc;
  const LevelInfo& L = p->L[level];
  DVO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  int info[2];
  DVO_CUDA(ctx, cudaMemcpy(info, p->sel_info + 2 * level, sizeof(info), cudaMemcpyDeviceToHost));
  if (count) *count = info[0];
  if (mask) {
    std::vector<uint32_t> words(L.words);
    DVO_CUDA(ctx, cudaMemcpy(words.data(), p->sel_mask + L.mask_off, sizeof(uint32_t) * L.words, cudaMemcpyDeviceToHost));
    for (int i = 0; i < L.n; ++i) mask[i] = (words[i >> 5] >> (i & 31)) & 1u;
  }
  return 0;
}

int dvo_b200_match_batch(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                         dvo_b200_pyramid* const* currents, const double* T_init, dvo_b200_result* results,
                         dvo_b200_iteration_stats* iteration_stats, int32_t max_iteration_stats) {
  if (!ctx || !results) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch: null argument");
  cudaSetDevice(ctx->device);
  MatchCall c;
  c.cfg = cfg; c.n = n; c.refs = references; c.curs = currents; c.T_init = T_init;
  c.results = results; c.iter_stats = iteration_stats; c.max_log = max_iteration_stats;
  return tracker_match(ctx, c);
}

int dvo_b200_match(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference, dvo_b200_pyramid* current,
                   const double* T_init, dvo_b200_result* result) {
  dvo_b200_pyramid* r[1] = {reference};
  dvo_b200_pyramid* c[1] = {current};
  return dvo_b200_match_batch(ctx, cfg, 1, r, c, T_init, result, nullptr, 0);
}

int dvo_b200_match_batch_device(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n,
                                dvo_b200_pyramid* const* references, dvo_b200_pyramid* const* currents,
                                const double* T_init, void* d_results) {
  if (!ctx || !d_results) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_device: null argument");
  cudaSetDevice(ctx->device);
  MatchCall c;
  c.cfg = cfg; c.n = n; c.refs = references; c.curs = currents; c.T_init = T_init;
  c.d_results = d_results;
  return tracker_match(ctx, c);
}

int dvo_b200_residual_image(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                            dvo_b200_pyramid* current, int32_t level, const double* T, float* planes7, int64_t* count) {
  if (!ctx || !cfg || !planes7) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "residual_image: null argument");
  cudaSetDevice(ctx->device);
  return tracker_linearize(ctx, cfg, reference, current, level, T, 0, nullptr, count, nullptr, nullptr, nullptr, nullptr, planes7);
}

int dvo_b200_intensity_error_image(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                                   dvo_b200_pyramid* current, int32_t level, const double* T, float* image, int64_t* count) {
  if (!ctx || !cfg || !image || !reference || !current) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "intensity_error_image: null argument");
  if (level < 0 || level >= reference->levels) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "intensity_error_image: level out of range");
  const size_t n = size_t(reference->L[level].w) * reference->L[level].h;
  std::vector<float> planes(7 * n);
  int64_t valid = 0;
  int rc = dvo_b200_residual_image(ctx, cfg, reference, current, level, T, planes.data(), &valid);
  if (rc != 0) return rc;
  // the residual stage leaves NaN at pixels that are unselected, dropped (odd last point, reference estimator) or invalid
  // after the warp: exactly the pixels the reference's raster walk leaves at the zero initialisation (dense_tracking.cpp:415-439)
  for (size_t i = 0; i < n; ++i) image[i] = planes[i] == planes[i] ? fabsf(planes[i]) : 0.0f;
  if (count) *count = valid;
  return 0;
}

int dvo_b200_linearize(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference, dvo_b200_pyramid* current,
                       int32_t level, const double* T, int32_t use_weights, const float* prev_precision, int64_t* count,
                       float* precision_out, float* ll_out, double* A_out, double* b_out) {
  if (!ctx || !cfg) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "linearize: null argument");
  cudaSetDevice(ctx->device);
  return tracker_linearize(ctx, cfg, reference, current, level, T, use_weights, prev_precision, count, precision_out, ll_out,
                           A_out, b_out, nullptr);
}

// ---- photometric mode ----
static bool all_finite(const double* v, size_t n) {
  for (size_t i = 0; i < n; ++i)
    if (!std::isfinite(v[i])) return false;
  return true;
}

int dvo_b200_match_batch_photometric(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                                     dvo_b200_pyramid* const* currents, const double* T_init, const double* photometric_init,
                                     dvo_b200_result* results, double* photometric, dvo_b200_iteration_stats* iteration_stats,
                                     int32_t max_iteration_stats) {
  if (!ctx || !results || !photometric) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_photometric: null argument");
  if (photometric_init && n > 0 && !all_finite(photometric_init, 2 * (size_t)n))
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_photometric: photometric_init is not finite");
  cudaSetDevice(ctx->device);
  MatchCall c;
  c.cfg = cfg; c.n = n; c.refs = references; c.curs = currents; c.T_init = T_init;
  c.ab_init = photometric_init;
  c.results = results; c.ab_out = photometric; c.iter_stats = iteration_stats; c.max_log = max_iteration_stats;
  return tracker_match(ctx, c);
}

// ---- motion prior ----
int dvo_b200_match_batch_prior(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                               dvo_b200_pyramid* const* currents, const double* T_init, const double* prior_information,
                               const double* photometric_init, double* photometric, dvo_b200_result* results,
                               dvo_b200_iteration_stats* iteration_stats, int32_t max_iteration_stats) {
  if (!ctx || !results) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_prior: null argument");
  const std::string why = prior_args_error(cfg, n, prior_information, photometric_init, photometric);
  if (!why.empty()) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, why);
  if (photometric_init && n > 0 && !all_finite(photometric_init, 2 * (size_t)n))
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_prior: photometric_init is not finite");
  cudaSetDevice(ctx->device);
  MatchCall c;
  c.cfg = cfg; c.n = n; c.refs = references; c.curs = currents; c.T_init = T_init;
  c.prior = prior_information; c.ab_init = photometric_init;
  c.results = results; c.ab_out = photometric; c.iter_stats = iteration_stats; c.max_log = max_iteration_stats;
  return tracker_match(ctx, c);
}

// ---- weight maps ----
// The largest extents of a batch's references at cfg->last_level and level 0, or false for a batch the match would refuse
// (the maps are then checked as for n = 0 and the batch checks refuse it)
static bool maps_extent(const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references, MapsExtent* ext) {
  *ext = MapsExtent{0, 0, 0, 0};
  if (!(cfg && n > 0 && references && cfg->last_level >= 0 && cfg->last_level < kMaxLevels)) return false;
  for (int32_t i = 0; i < n; ++i) {
    const dvo_b200_pyramid* r = references[i];
    if (!r || r->levels <= cfg->last_level) return false;
    ext->w = std::max(ext->w, r->L[cfg->last_level].w); ext->h = std::max(ext->h, r->L[cfg->last_level].h);
    ext->w0 = std::max(ext->w0, r->L[0].w); ext->h0 = std::max(ext->h0, r->L[0].h);
  }
  return true;
}

// where one byte of a maps output lies (maps_args.h)
static PtrWhere pointer_where(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return PtrWhere{kPtrHost, -1}; }
  if (a.type == cudaMemoryTypeDevice) return PtrWhere{kPtrDevice, a.device};
  if (a.type == cudaMemoryTypeManaged) return PtrWhere{kPtrManaged, a.device};
  return PtrWhere{kPtrHost, -1};
}

int dvo_b200_match_batch_maps(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                              dvo_b200_pyramid* const* currents, const double* T_init, const double* prior_information,
                              const double* photometric_init, double* photometric, dvo_b200_result* results,
                              dvo_b200_iteration_stats* iteration_stats, int32_t max_iteration_stats, const dvo_b200_weight_maps* maps) {
  if (!ctx || !results) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_maps: null argument");
  // the refusals of the entry point without maps that come before its batch checks
  if (prior_information) {
    const std::string why = prior_args_error(cfg, n, prior_information, photometric_init, photometric);
    if (!why.empty()) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, why);
  } else if (photometric_init && !photometric) {
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_maps: photometric_init without photometric");
  }
  if (photometric_init && n > 0 && !all_finite(photometric_init, 2 * (size_t)n))
    return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_maps: photometric_init is not finite");
  cudaSetDevice(ctx->device);
  MapsExtent ext;
  const bool sane = maps_extent(cfg, n, references, &ext);
  const std::string why = maps_args_error(maps, sane ? n : 0, ext, ctx->device, pointer_where);
  if (!why.empty()) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, why);
  MatchCall c;
  c.cfg = cfg; c.n = n; c.refs = references; c.curs = currents; c.T_init = T_init;
  c.prior = prior_information; c.ab_init = photometric_init;
  c.results = results; c.ab_out = photometric; c.iter_stats = iteration_stats; c.max_log = max_iteration_stats; c.maps = maps;
  return tracker_match(ctx, c);
}

// ---- multi-hypothesis alignment ----
int dvo_b200_match_batch_hypotheses_modes(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                                          dvo_b200_pyramid* const* currents, int32_t k, const double* hypotheses, int32_t screen_level,
                                          double min_constraint_ratio, const double* prior_information, const double* photometric_init,
                                          double* photometric, double* screen_photometric, dvo_b200_result* results, int32_t* best,
                                          double* scores, dvo_b200_result* screen_results, dvo_b200_iteration_stats* iteration_stats,
                                          int32_t max_iteration_stats, const dvo_b200_weight_maps* maps) {
  if (!ctx) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "match_batch_hypotheses: null argument");
  MapsExtent ext;
  const bool sane = maps && maps_extent(cfg, n, references, &ext);
  const std::string why = hypotheses_modes_args_error(cfg, n, k, hypotheses, screen_level, min_constraint_ratio, results, best,
                                                      prior_information, photometric_init, photometric, screen_photometric, maps,
                                                      sane ? &ext : nullptr, ctx->device, pointer_where);
  if (!why.empty()) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, why);
  cudaSetDevice(ctx->device);
  MatchCall c;
  c.cfg = cfg; c.n = n; c.refs = references; c.curs = currents; c.T_init = hypotheses;
  c.k = k; c.screen_level = screen_level; c.min_ratio = min_constraint_ratio;
  c.prior = prior_information; c.ab_init = photometric_init;
  c.results = results; c.ab_out = photometric; c.screen_ab = screen_photometric;
  c.best = best; c.scores = scores; c.screen_results = screen_results;
  c.iter_stats = iteration_stats; c.max_log = max_iteration_stats; c.maps = maps;
  return tracker_match(ctx, c);
}

int dvo_b200_match_batch_hypotheses(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, int32_t n, dvo_b200_pyramid* const* references,
                                    dvo_b200_pyramid* const* currents, int32_t k, const double* hypotheses, int32_t screen_level,
                                    double min_constraint_ratio, dvo_b200_result* results, int32_t* best, double* scores,
                                    dvo_b200_result* screen_results, dvo_b200_iteration_stats* iteration_stats,
                                    int32_t max_iteration_stats) {
  return dvo_b200_match_batch_hypotheses_modes(ctx, cfg, n, references, currents, k, hypotheses, screen_level, min_constraint_ratio,
                                               nullptr, nullptr, nullptr, nullptr, results, best, scores, screen_results,
                                               iteration_stats, max_iteration_stats, nullptr);
}

int dvo_b200_residual_image_photometric(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                                        dvo_b200_pyramid* current, int32_t level, const double* T, const double ab[2], float* planes7,
                                        int64_t* count) {
  if (!ctx || !cfg || !planes7 || !ab) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "residual_image_photometric: null argument");
  if (!all_finite(ab, 2)) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "residual_image_photometric: ab is not finite");
  cudaSetDevice(ctx->device);
  return tracker_linearize(ctx, cfg, reference, current, level, T, 0, nullptr, count, nullptr, nullptr, nullptr, nullptr, planes7, ab);
}

int dvo_b200_linearize_photometric(dvo_b200_ctx* ctx, const dvo_b200_config* cfg, dvo_b200_pyramid* reference,
                                   dvo_b200_pyramid* current, int32_t level, const double* T, const double ab[2], int32_t use_weights,
                                   const float* prev_precision, int64_t* count, float* precision_out, float* ll_out, double* A_out,
                                   double* b_out) {
  if (!ctx || !cfg || !ab) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "linearize_photometric: null argument");
  if (!all_finite(ab, 2)) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "linearize_photometric: ab is not finite");
  cudaSetDevice(ctx->device);
  return tracker_linearize(ctx, cfg, reference, current, level, T, use_weights, prev_precision, count, precision_out, ll_out,
                           A_out, b_out, nullptr, ab);
}

int dvo_b200_profile_enable(dvo_b200_ctx* ctx, int32_t enable) {
  if (!ctx) return DVO_B200_ERR_INVALID_ARGUMENT;
  ctx->profile = enable != 0;
  return 0;
}

int dvo_b200_profile_read(dvo_b200_ctx* ctx, double ms_out[8], int64_t launches_out[8], int32_t reset) {
  if (!ctx) return DVO_B200_ERR_INVALID_ARGUMENT;
  cudaSetDevice(ctx->device);
  drain_profile(ctx);
  if (ctx->d_dbg) {   // developer timing dump (DVO_B200_TIMING=1)
    unsigned long long h[256];
    cudaStreamSynchronize(ctx->stream);
    cudaMemcpy(h, ctx->d_dbg, sizeof(h), cudaMemcpyDeviceToHost);
    static const char* names[8] = {"stageA", "stageB", "waitA", "waitB", "mid", "end", "queue", "total"};
    for (int l = 0; l < 8; ++l) {
      const unsigned long long* v = h + 16 * l;
      if (!v[7]) continue;
      fprintf(stderr, "[dvo_b200 timing] level-slot %d:", l);
      for (int i = 0; i < 8; ++i) fprintf(stderr, " %s=%.1f%%", names[i], 100.0 * (double)v[i] / (double)v[7]);
      fprintf(stderr, " (cta-ms total %.1f)\n", (double)v[7] * 1e-6);
      fprintf(stderr, "[dvo_b200 timing]   consumer warp 0: wait-full %.1f%% of stage A, %.1f%% of stage B; producer: descriptor %.1f%%, "
                      "wait-empty %.1f%% of its stage time\n", 100.0 * (double)v[9] / (double)(v[8] + 1), 100.0 * (double)v[11] / (double)(v[10] + 1),
              100.0 * (double)v[12] / (double)(v[14] + v[15] + 1), 100.0 * (double)v[13] / (double)(v[14] + v[15] + 1));
      const unsigned long long* u = h + 128 + 8 * l;
      if (u[0]) fprintf(stderr, "[dvo_b200 timing]   tiles %llu (inexact %.2f%%, skipped %.2f%%), stage-B rounds in the generic loop %.2f%%; CTA lifetime of the last launch-set: "
                                "max %.3f ms, min %.3f ms\n", u[0], 100.0 * (double)u[1] / (double)u[0], 100.0 * (double)u[2] / (double)u[0],
                        100.0 * (double)u[4] / (double)(u[3] + 1), (double)u[5] * 1e-6, (double)u[6] * 1e-6);
      if (u[7]) fprintf(stderr, "[dvo_b200 timing]   cmask tiles %llu (%.2f%% of all tiles): stage-B tiles that test the current image's mask "
                                "per tap\n", u[7], 100.0 * (double)u[7] / (double)(u[0] + 1));
      const unsigned long long* e = h + 192 + 8 * l;   // e[7]: critical ns; e[0..5]: sub-phases
      if (e[7]) {
        double tot = 0;
        for (int i = 0; i < 6; ++i) tot += (double)e[i];
        fprintf(stderr, "[dvo_b200 timing]   end step: critical part %.1f%% of the end time; of the end thread's time: partial sums %.1f%%, state+log %.1f%%, "
                        "LDLT %.1f%%, exp+K*T %.1f%%, release %.1f%%, deferred %.1f%% (total %.1f cta-ms)\n", 100.0 * (double)e[7] / (double)(v[5] + 1),
                100.0 * e[0] / tot, 100.0 * e[1] / tot, 100.0 * e[2] / tot, 100.0 * e[3] / tot, 100.0 * e[4] / tot, 100.0 * e[5] / tot, tot * 1e-6);
      }
    }
    if (reset) {
      cudaMemset(ctx->d_dbg, 0, sizeof(h));
      for (int l = 0; l < 8; ++l) { unsigned long long big = ~0ull; cudaMemcpy(ctx->d_dbg + 128 + 8 * l + 6, &big, 8, cudaMemcpyHostToDevice); }
    }
  }
  if (getenv("DVO_B200_TIMING")) {   // developer: device time of the level kernels, per level of the match (coarse -> fine)
    fprintf(stderr, "[dvo_b200 timing] level kernels, ms per launch:");
    for (int i = 8; i < 16; ++i)
      if (ctx->prof_launches[i]) fprintf(stderr, " %.3f", ctx->prof_ms[i] / (double)ctx->prof_launches[i]);
    fprintf(stderr, "\n");
  }
  for (int i = 0; i < 16; ++i) {
    if (i < 8 && ms_out) ms_out[i] = ctx->prof_ms[i];
    if (i < 8 && launches_out) launches_out[i] = ctx->prof_launches[i];
    if (reset) { ctx->prof_ms[i] = 0; ctx->prof_launches[i] = 0; }
  }
  return 0;
}

}  // extern "C"
