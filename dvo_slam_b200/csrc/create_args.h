// create_args.h -- one pyramid create as its entry point was called, and every check of it that needs no CUDA call: the
// arguments, the rectifier, the depth registration and the level geometry.  Plain C++ without CUDA, so that the checks can
// be built and run on the host alone (tests/native/create_args.cpp).  capi.cu runs them before any upload or launch, then
// checks the dvo_b200_device_planes of a device create.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

#include "../../include/dvo_b200.h"

struct dvo_b200_rectifier {      // a remap to a pinhole camera (dvo_b200_rectifier_create)
  dvo_b200_ctx* ctx = nullptr;   // the owning context: its stream orders every use and the free
  int in_w = 0, in_h = 0;        // input frames
  int w = 0, h = 0;              // rectified frames = level 0
  float K[4] = {0, 0, 0, 0};     // K_new: fx, fy, cx, cy of level 0
  float* map = nullptr;          // device, stream-ordered allocation: map_x[w*h] then map_y[w*h]
};

struct dvo_b200_depth_registration {   // a depth camera reprojected into a pinhole colour camera (dvo_b200_depth_registration_create)
  dvo_b200_ctx* ctx = nullptr;          // the owning context: its stream orders every use and the free
  int dw = 0, dh = 0;                   // depth frames
  int w = 0, h = 0;                     // colour frames = level 0
  float R[9] = {}, t[3] = {};           // T_color_depth, each value rounded once
  float K[4] = {0, 0, 0, 0};            // fx, fy, cx, cy of level 0
  float* rays = nullptr;                // device, stream-ordered: cx_ray, cy_ray [dw*dh] then kx_ray, ky_ray [(dw+1)*(dh+1)]
};

namespace dvo_b200 {

constexpr int kMaxLevels = DVO_B200_MAX_LEVELS;

// tile geometry of the level kernel (tracker.cu) and of the per-tile depth ranges (pyramid.cu)
constexpr int kTileW = 160;    // reference pixels per tile row: 5 warp rounds; 640, 320 and 160 columns are whole bands
#ifndef DVO_TILE_H
#define DVO_TILE_H 7
#endif
constexpr int kTileH = DVO_TILE_H;      // tile rows = consumer warps of a CTA (warp q walks row q of every tile of a strip); 7 consumers +
                               // 1 producer warp = 256 threads, two CTAs per SM at 128 registers per thread

// ---- device image layout --------------------------------------------------------------------
// Per image, per level l: two float2 planes of h_l rows, row pitch = w_l rounded up to even (every row
// starts 16-byte aligned, which the bulk-copy engine requires of its sources), for the role of CURRENT image:
//   P0 = (I, Z')   P2 = (I, Z)
// and the REFERENCE TILE RECORDS (common.cuh) for the role of reference image: (I, Zsel), tx and (Ix, Iy) per tile.
// Z' is the depth with NaN wherever ANY of the six channels is NaN at that pixel: a bilinear tap
// on such a pixel makes the reference reject the point (cmpunord over the 8-vector,
// dense_tracking_impl.cpp:261) and a reference point there fails isPointOk (point_selection.h:63-66),
// so one NaN test on the interpolated Z' replaces the reference's test on all lanes.
// The 8-channel AoS "acceleration" image of the reference (rgbd_image.cpp:534-543) exists only to
// make CPU gathers contiguous.  The tracker stages rectangular windows of ONE float2 plane of the
// current image in shared memory: P0 for the residual/weight/scale stage, P2 (true depth) for the
// linearisation stage, which forms the four gradient channels of every bilinear tap from the staged
// (I, Z) neighbours with the very operations of calculateDerivativeX/Y (rgbd_image.cpp:419-472), so
// gradient planes of the current image are never read (the depth gradients are not even stored).
// Zsel is the depth where the pixel belongs to the reference point list of PointSelection::select
// (point_selection.cpp:89-152; the odd last point that computeResidualsSse skips excluded) and NaN
// elsewhere: the reference side of an alignment reads the tile records and needs no mask lookup -- an
// unselected point projects to NaN and fails the bounds test like any other rejected point.
struct LevelInfo {
  int w, h, n, words;          // n = w*h pixels, words = ceil(n/32) selection-mask words (linear index y*w+x)
  int pitch;                   // row pitch of the planes in float2 elements (w rounded up to even)
  int nbands, nstrips;         // tiles of kTileW x kTileH reference pixels: nbands x nstrips
  float fx, fy, ox, oy;        // IntrinsicMatrix of this level (intrinsic_matrix.cpp:90-93: whole K * 0.5)
  size_t plane_off;            // float2 offset of P0 = (I, Z') inside dvo_b200_pyramid::planes; P2 = (I, Z) follows at + pitch*h
  size_t rec_off;              // float2 offset of the reference tile records (kRecF2 each, tile = strip * nbands + band)
  size_t mask_off;             // uint32 offset inside sel_mask
  size_t tmpl_off;             // float offset of tx[w] then ty[h] inside tmpl
  size_t range_off;            // float2 offset of the per-tile depth range {zmin, zmax} inside tile_range
  size_t sat_off;              // int offset of the unusable-pixel summary inside cur_sat (BOTH pyramids only)
};

inline std::string size_str(int w, int h) { return std::to_string(w) + "x" + std::to_string(h); }

// The levels of a pyramid whose level 0 is w x h pixels with intrinsics K = fx, fy, ox, oy: the sizes, intrinsics and tile
// counts of L[0 .. levels) (the slab offsets are the build's).  Returns "" or why the geometry is refused.
inline std::string derive_levels(int w, int h, const float K[4], int levels, LevelInfo* L) {
  if (levels < 1 || levels > kMaxLevels) return "levels " + std::to_string(levels) + " outside 1.." + std::to_string(kMaxLevels);
  if (w < 32 || h < 2) return "level 0 of " + size_str(w, h) + " is below 32 wide or 2 high";
  for (int l = 0; l < levels; ++l) {
    LevelInfo& q = L[l];
    if (l == 0) { q.w = w; q.h = h; q.fx = K[0]; q.fy = K[1]; q.ox = K[2]; q.oy = K[3]; }
    else {
      q.w = L[l - 1].w / 2; q.h = L[l - 1].h / 2;
      q.fx = L[l - 1].fx * 0.5f; q.fy = L[l - 1].fy * 0.5f; q.ox = L[l - 1].ox * 0.5f; q.oy = L[l - 1].oy * 0.5f;
    }
    // odd sizes: the last column / row is dropped by the 2x2 mean exactly as in pyrDownMeanSmooth (rgbd_image.cpp:41)
    if (q.w < 8 || q.h < 2) return "level " + std::to_string(l) + " of " + size_str(q.w, q.h) + " is below 8x2";
    // the level kernel splits a linear pixel index with one multiply-high (tracker.cu): exact only below this bound
    if ((uint64_t)q.w * q.h >= (1ull << 30)) return "level " + std::to_string(l) + " of " + size_str(q.w, q.h) + " has 2^30 pixels or more";
    q.n = q.w * q.h;
    q.words = (q.n + 31) / 32;
    q.pitch = (q.w + 1) & ~1;
    q.nbands = (q.w + kTileW - 1) / kTileW;
    q.nstrips = (q.h + kTileH - 1) / kTileH;
  }
  return "";
}

// What the level-0 planes go through before the build
enum CreateRemap { kRemapNone, kRemapRectify, kRemapRegister };

// One create call.  The host forms set image / depth / masks, the device forms (device = true) the three planes; masks NULL:
// no mask, whatever the roles.  K: level 0's intrinsics without a rectifier or registration, which bring their own.
struct CreateArgs {
  const char* fn = "";                               // the entry point, the prefix of its errors
  int n = 0, format = DVO_B200_INPUT_FLOAT32;
  float depth_scale = 0.f;
  int roles = DVO_B200_MASK_ROLE_REFERENCE, width = 0, height = 0;
  float K[4] = {0, 0, 0, 0};
  int levels = 0;
  int remap = kRemapNone;
  const dvo_b200_rectifier* rect = nullptr;           // required by kRemapRectify, optional with kRemapRegister
  const dvo_b200_depth_registration* reg = nullptr;   // required by kRemapRegister
  bool device = false;
  const void* image = nullptr;
  const void* depth = nullptr;
  const uint8_t* masks = nullptr;
  const dvo_b200_device_plane* image_plane = nullptr;
  const dvo_b200_device_plane* depth_plane = nullptr;
  const dvo_b200_device_plane* mask_plane = nullptr;
};

// Level 0 of the build: the registration's or the rectifier's target and K, else the frames and a.K.
inline void create_level0(const CreateArgs& a, int* w, int* h, const float** K) {
  if (a.reg) { *w = a.reg->w; *h = a.reg->h; *K = a.reg->K; }
  else if (a.rect) { *w = a.rect->w; *h = a.rect->h; *K = a.rect->K; }
  else { *w = a.width; *h = a.height; *K = a.K; }
}

// Every check of a create that needs no CUDA call, in this order: ctx and the null / size arguments, the format, the roles,
// the rectifier, the depth registration, the level geometry.  Returns "" or the refusal, prefixed with a.fn.
inline std::string create_args_error(const dvo_b200_ctx* ctx, const CreateArgs& a, const void* out) {
  auto bad = [&](const std::string& why) { return std::string(a.fn) + ": " + why; };
  const bool frames = a.device ? a.image_plane && a.depth_plane : a.image && a.depth;
  if (!ctx || !frames || !out || a.n <= 0 || a.width <= 0 || a.height <= 0) return bad("null/invalid argument");
  if (a.format != DVO_B200_INPUT_FLOAT32 && a.format != DVO_B200_INPUT_GREY8_DEPTH16 && a.format != DVO_B200_INPUT_BGR8_DEPTH16)
    return bad("unknown input format " + std::to_string(a.format));
  if (a.roles != DVO_B200_MASK_ROLE_REFERENCE && a.roles != (DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT))
    return bad("unsupported role set " + std::to_string(a.roles));
  if (a.remap == kRemapRectify || a.rect) {
    if (!a.rect) return bad("null rectifier");
    if (a.rect->ctx != ctx) return bad("the rectifier belongs to another context");
    if (a.width != a.rect->in_w || a.height != a.rect->in_h)
      return bad("frames of " + size_str(a.width, a.height) + ", the rectifier takes " + size_str(a.rect->in_w, a.rect->in_h));
  }
  if (a.remap == kRemapRegister) {
    const dvo_b200_depth_registration* reg = a.reg;
    if (!reg) return bad("null depth registration");
    if (reg->ctx != ctx) return bad("the depth registration belongs to another context");
    if (a.rect) {
      if (a.rect->w != reg->w || a.rect->h != reg->h)
        return bad("the rectifier's output is not the registration's target " + size_str(reg->w, reg->h));
      for (int i = 0; i < 4; ++i)
        if (a.rect->K[i] != reg->K[i]) return bad("the rectifier's K_new is not the registration's K");
    } else if (a.width != reg->w || a.height != reg->h) {
      return bad("colour frames of " + size_str(a.width, a.height) + ", the registration's target is " + size_str(reg->w, reg->h));
    }
  }
  int w, h;
  const float* K;
  create_level0(a, &w, &h, &K);
  LevelInfo L[kMaxLevels];
  const std::string why = derive_levels(w, h, K, a.levels, L);
  return why.empty() ? why : bad(why);
}

}  // namespace dvo_b200
