// pyramid.cu -- device image pyramid: replaces RgbdImagePyramid::build (rgbd_image.cpp:156-172),
// pyrDownMeanSmooth / pyrDownSubsample (rgbd_image.cpp:38-55,127-139), RgbdCameraPyramid::build
// (rgbd_image.cpp:283-296), calculateDerivativeX/Y (rgbd_image.cpp:419-472, rgbd_image_sse.cpp:241-284),
// the RgbdCamera point-cloud template (rgbd_image.cpp:186-204) and PointSelection::select with the
// default predicate (point_selection.cpp:89-152, point_selection.h:63-66).
#include "common.cuh"

#include <cstdio>
#include <cstring>

namespace dvo_b200 {

namespace {

__device__ __forceinline__ bool is_nan(float v) { return v != v; }

// Level-0 pixels as the caller's planes hold them (uploaded into staging, or in place in the caller's device memory; i is
// the element index of a SrcPlane).  kRaw = false: float32 intensity and float32 depth in metres (NaN = invalid), what
// benchmark_slam.cpp:46-93 hands to RgbdCameraPyramid::create.  kRaw = true: 8-bit grey and 16-bit raw depth straight from
// the image files; the loader's conversions -- convertTo(CV_32F) and SurfacePyramid::convertRawDepthImageSse
// (surface_pyramid.cpp:65-105: u16 * scale, 0 -> NaN) -- happen in the load, no float32 copy of the frame is ever written.
template <bool kRaw>
__device__ __forceinline__ float load_intensity(const void* I, size_t i) {
  if (kRaw) return (float)__ldg(reinterpret_cast<const uint8_t*>(I) + i);
  return __ldg(reinterpret_cast<const float*>(I) + i);
}
template <bool kRaw>
__device__ __forceinline__ float load_depth(const void* Z, size_t i, float scale) {
  if (kRaw) {
    const uint16_t r = __ldg(reinterpret_cast<const uint16_t*>(Z) + i);
    return r == 0 ? __int_as_float(0x7fc00000) : __fmul_rn((float)r, scale);
  }
  return __ldg(reinterpret_cast<const float*>(Z) + i);
}

// level l intensity = ((a+b)+c)+d)/4 of the 2x2 block of level l-1 (rgbd_image.cpp:38-55), into P0.x (the Z slot is
// filled by the finish pass).  kFromInput: level 1 reads the input plane I0, which is level 0's intensity.  aligned: the
// base address, row pitch and image stride of I0 are all multiples of two elements, so every 2x2 block starts at a
// two-element boundary (packed planes: even w and w*h).  sp / dp: row pitch of the source / destination planes (float2
// elements).
template <bool kFromInput, bool kRaw>
__global__ void k_pyr_intensity_down(SrcPlane I0, int aligned, float2* __restrict__ planes, size_t planes_per_image,
                                     size_t src_off, int sp, size_t dst_off, int dw, int dh, int dp) {
  int img = blockIdx.y;
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= dw * dh) return;
  int y = idx / dw, x = idx - y * dw;
  float2* D = planes + img * planes_per_image + dst_off;
  float a, b, c, d;
  if (kFromInput) {
    const size_t i0 = I0.at(img, 2 * y, 2 * x);
    const int64_t r = I0.pitch;
    if (kRaw) {
      const uint8_t* g = reinterpret_cast<const uint8_t*>(I0.data) + i0;
      if (aligned) {
        const uchar2 u = __ldg(reinterpret_cast<const uchar2*>(g)), v = __ldg(reinterpret_cast<const uchar2*>(g + r));
        a = (float)u.x; b = (float)u.y; c = (float)v.x; d = (float)v.y;
      } else {
        a = (float)__ldg(g); b = (float)__ldg(g + 1); c = (float)__ldg(g + r); d = (float)__ldg(g + r + 1);
      }
    } else {
      const float* p0 = reinterpret_cast<const float*>(I0.data) + i0;
      if (aligned) {
        const float2 u = __ldg(reinterpret_cast<const float2*>(p0)), v = __ldg(reinterpret_cast<const float2*>(p0 + r));
        a = u.x; b = u.y; c = v.x; d = v.y;
      } else {
        a = __ldg(p0); b = __ldg(p0 + 1); c = __ldg(p0 + r); d = __ldg(p0 + r + 1);
      }
    }
  } else {
    const float2* S = planes + img * planes_per_image + src_off;
    const float2* r0 = S + (size_t)(2 * y) * sp + 2 * x;
    const float2* r1 = r0 + sp;
    a = r0[0].x; b = r0[1].x; c = r1[0].x; d = r1[1].x;
  }
  float s = __fadd_rn(a, b);
  s = __fadd_rn(s, c);
  s = __fadd_rn(s, d);
  D[(size_t)y * dp + x] = make_float2(s * 0.25f, 0.f);
}

__device__ __forceinline__ bool bit_set(const uint32_t* __restrict__ words, size_t i) { return (__ldg(words + (i >> 5)) >> (i & 31)) & 1u; }

// Usable bits of one level of a pyramid built with a reference mask, in the word layout of the selection masks (bit i of
// word k = linear pixel 32k+i).  Level 0: the caller's mask plane of bytes, nonzero = usable.  Level l: a pixel is usable
// iff the four pixels of its 2x2 block in level l-1 are -- the chain of the 2x2 intensity mean -- so iff every level-0 pixel
// of its footprint [x 2^l, (x+1) 2^l) x [y 2^l, (y+1) 2^l) is.  Runs before k_pyr_finish of the same level.
template <bool kLevel0>
__global__ void __launch_bounds__(256)
k_usable(SrcPlane mask0, uint32_t* __restrict__ usable, size_t words_per_image, size_t src_off, int sw, size_t dst_off, int w,
         int h) {
  const int img = blockIdx.y;
  const int n = w * h;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t* U = usable + img * words_per_image;
  bool u = false;
  if (idx < n) {
    if (kLevel0) {   // rows packed (the staged masks): the linear index needs no division
      const size_t i = mask0.pitch == w ? (size_t)((int64_t)img * mask0.stride) + idx : mask0.at(img, idx / w, idx % w);
      u = __ldg(reinterpret_cast<const uint8_t*>(mask0.data) + i) != 0;
    } else {
      const int y = idx / w, x = idx - y * w;
      const size_t j = (size_t)(2 * y) * sw + 2 * x;   // top-left pixel of the block in level l-1
      const uint32_t* S = U + src_off;
      u = bit_set(S, j) && bit_set(S, j + 1) && bit_set(S, j + sw) && bit_set(S, j + sw + 1);
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, u);
  if ((threadIdx.x & 31) == 0 && idx < ((n + 31) / 32) * 32) U[dst_off + (idx >> 5)] = m;
}

// gradients (clamped central differences), masked and true depth, default selection mask and reference plane
// (I, Zsel: depth where the pixel is selected, NaN elsewhere) for one level.
// Depth of level l is the pure subsample chain of level 0 (rgbd_image.cpp:127-139): Z_l(y,x) = Z_0(y<<l, x<<l).
// Level 0 reads its intensity straight from the input image I0 (no intermediate copy); the other levels read the
// intensity that k_pyr_intensity_down left in P0.x.  The selection count / last selected index are derived from
// the masks afterwards (k_sel_info): no atomics here.  Threads walk the linear pixel index y*w+x (the order of the
// selection mask); the planes are addressed with the row pitch.  kMasked: the selection also requires the pixel's usable
// bit (k_usable); only the reference role changes, P0 / P2 are written as without a mask.
template <bool kLevel0, bool kRaw, bool kMasked>
__global__ void __launch_bounds__(256)
k_pyr_finish(SrcPlane I0, SrcPlane Z0, float zscale, float2* __restrict__ planes, size_t planes_per_image, size_t plane_off,
             size_t rec_off, int nbands, int w, int h, int pitch, int level, uint32_t* __restrict__ masks,
             size_t mask_words_per_image, size_t mask_off, float ti, float td, const uint32_t* __restrict__ usable) {
  const int img = blockIdx.y;
  const int n = w * h;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = idx < n;
  bool sel = false;
  if (in) {
    const int y = idx / w, x = idx - y * w;
    const size_t plane = (size_t)pitch * h;
    float2* P0 = planes + img * planes_per_image + plane_off;
    float2* P2 = P0 + plane;   // P2 = (I, Z); the depth gradients are not stored
    float2* rec = planes + img * planes_per_image + rec_off;   // reference tile records: (I, Zsel) and (Ix, Iy)
    const int xp = max(x - 1, 0), xn = min(x + 1, w - 1), yp = max(y - 1, 0), yn = min(y + 1, h - 1);
    float I, ixp, ixn, iyp, iyn;
    if (kLevel0) {
      const void* g = I0.data;
      I = load_intensity<kRaw>(g, I0.at(img, y, x)); ixp = load_intensity<kRaw>(g, I0.at(img, y, xp));
      ixn = load_intensity<kRaw>(g, I0.at(img, y, xn));
      iyp = load_intensity<kRaw>(g, I0.at(img, yp, x)); iyn = load_intensity<kRaw>(g, I0.at(img, yn, x));
    } else {
      const size_t row = (size_t)y * pitch;
      I = P0[row + x].x; ixp = P0[row + xp].x; ixn = P0[row + xn].x;
      iyp = P0[(size_t)yp * pitch + x].x; iyn = P0[(size_t)yn * pitch + x].x;
    }
    const float ix = (ixn - ixp) * 0.5f;
    const float iy = (iyn - iyp) * 0.5f;
    const void* zp = Z0.data;
    const float z = load_depth<kRaw>(zp, Z0.at(img, y << level, x << level), zscale);
    const float zx = (load_depth<kRaw>(zp, Z0.at(img, y << level, xn << level), zscale) -
                      load_depth<kRaw>(zp, Z0.at(img, y << level, xp << level), zscale)) * 0.5f;
    const float zy = (load_depth<kRaw>(zp, Z0.at(img, yn << level, x << level), zscale) -
                      load_depth<kRaw>(zp, Z0.at(img, yp << level, x << level), zscale)) * 0.5f;
    const bool bad = is_nan(I) || is_nan(ix) || is_nan(iy) || is_nan(z) || is_nan(zx) || is_nan(zy);
    const float zm = bad ? __int_as_float(0x7fc00000) : z;
    const size_t o = (size_t)y * pitch + x;
    // ValidPointAndGradientThresholdPredicate::isPointOk (point_selection.h:63-66)
    sel = !bad && (fabsf(ix) > ti || fabsf(iy) > ti || fabsf(zx) > td || fabsf(zy) > td);
    if (kMasked) sel = sel && bit_set(usable + img * mask_words_per_image + mask_off, idx);
    const float nanv = __int_as_float(0x7fc00000);
    const size_t rc = rec_cell(x, y, nbands);
    P0[o] = make_float2(I, zm);
    P2[o] = make_float2(I, z);
    rec[rc] = make_float2(I, sel ? z : nanv);
    rec[rc + kRecP1] = make_float2(ix, iy);
    if (x == w - 1 && pitch > w) {   // the pad column of an odd width: never a valid tap
      P0[o + 1] = make_float2(0.f, nanv);
      P2[o + 1] = make_float2(0.f, nanv);
    }
  }
  const unsigned m = __ballot_sync(0xffffffffu, sel);
  if ((threadIdx.x & 31) == 0 && idx < ((n + 31) / 32) * 32) masks[img * mask_words_per_image + mask_off + (idx >> 5)] = m;
}

// The parts of the reference tile records that no pixel owns: the tx[] slice of every tile and, in border tiles, the cells
// outside the image (never selected).  One thread per tile column; runs after k_template.
__global__ void k_rec_fill(float2* __restrict__ planes, size_t planes_per_image, size_t rec_off, int nbands, int ntiles, int w, int h,
                           const float* __restrict__ tmpl, size_t tmpl_per_image, size_t tmpl_off) {
  const int img = blockIdx.y;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ntiles * kTileW) return;
  const int tile = t / kTileW, cx = t - tile * kTileW;
  const int s = tile / nbands, b = tile - s * nbands;
  const int x = b * kTileW + cx, y0 = s * kTileH;
  float2* rec = planes + img * planes_per_image + rec_off + (size_t)tile * kRecF2;
  reinterpret_cast<float*>(rec + kRecTx)[cx] = x < w ? tmpl[img * tmpl_per_image + tmpl_off + x] : 0.f;
  const int r0 = x >= w ? 0 : min(max(h - y0, 0), kTileH);      // first row of this column that lies outside the image
  for (int r = r0; r < kTileH; ++r) {
    rec[r * kTileW + cx] = make_float2(0.f, __int_as_float(0x7fc00000));
    rec[kRecP1 + r * kTileW + cx] = make_float2(0.f, 0.f);
  }
}

// {min, max} of the non-NaN Z' of every tile of kTileW x kTileH pixels (one warp per tile).  The level kernel
// projects the tile's corner rays at both depths to bound the window of the current image its taps fall into.
// kMasked: only usable pixels count.  Every selected point, for any thresholds and the corrected estimator's odd point
// included, is usable with a non-NaN Z', so the range still covers them; a tile without usable depth is skipped.
template <bool kMasked>
__global__ void k_tile_range(const float2* __restrict__ planes, size_t planes_per_image, size_t plane_off, int w, int h,
                             int pitch, int nbands, int ntiles, float2* __restrict__ ranges, size_t ranges_per_image,
                             size_t range_off, const uint32_t* __restrict__ usable, size_t usable_per_image, size_t usable_off) {
  const int img = blockIdx.y;
  const int tile = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tile >= ntiles) return;
  const int lane = threadIdx.x & 31;
  const int s = tile / nbands, b = tile - s * nbands;
  const float2* P0 = planes + img * planes_per_image + plane_off;
  float lo = 3.0e38f, hi = -3.0e38f;
  const int x0 = b * kTileW, x1 = min(x0 + kTileW, w), y0 = s * kTileH, y1 = min(y0 + kTileH, h);
  for (int y = y0; y < y1; ++y)
    for (int x = x0 + lane; x < x1; x += 32) {
      const float z = P0[(size_t)y * pitch + x].y;
      if (kMasked && !bit_set(usable + img * usable_per_image + usable_off, (size_t)y * w + x)) continue;
      if (z == z) { lo = fminf(lo, z); hi = fmaxf(hi, z); }
    }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, off));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, off));
  }
  if (lane == 0) ranges[img * ranges_per_image + range_off + tile] = make_float2(lo, hi);
}

// Masks that also act in the CURRENT role, one level, after k_pyr_finish: one thread per kSatBlock x kSatBlock block writes
// Z' = NaN into P0 at the block's unusable pixels -- the residual stage then rejects any point with an unusable bilinear
// tap through its NaN test on the blended Z', as for a NaN depth -- and stores the block's unusable count into the
// summary (cell (by + 1, bx + 1), summed up by k_cur_sat).  P2 keeps the true (I, Z), so the gradients of usable taps
// next to an excluded region are those of the unmasked build.  Nothing else reads Z' at an unusable pixel: the selection,
// the tile depth ranges and the odd last point only look at usable pixels, and the next level's intensity reads P0.x.
__global__ void __launch_bounds__(256)
k_cur_mask(float2* __restrict__ planes, size_t planes_per_image, size_t plane_off, int w, int h, int pitch,
           const uint32_t* __restrict__ usable, size_t usable_per_image, size_t usable_off, int* __restrict__ sat,
           size_t sat_per_image, size_t sat_off) {
  const int img = blockIdx.y;
  const int cols = sat_cols(w) - 1, rows = sat_rows(h) - 1;
  const int blk = blockIdx.x * blockDim.x + threadIdx.x;
  if (blk >= cols * rows) return;
  const int by = blk / cols, bx = blk - by * cols;
  float2* P0 = planes + img * planes_per_image + plane_off;
  const uint32_t* U = usable + img * usable_per_image + usable_off;
  const int x0 = bx * kSatBlock, y0 = by * kSatBlock;
  const int x1 = min(x0 + kSatBlock, w), y1 = min(y0 + kSatBlock, h);
  int cnt = 0;
  for (int y = y0; y < y1; ++y)
    for (int x = x0; x < x1; ++x)
      if (!bit_set(U, (size_t)y * w + x)) {
        ++cnt;
        P0[(size_t)y * pitch + x].y = __int_as_float(0x7fc00000);
      }
  sat[img * sat_per_image + sat_off + (size_t)(by + 1) * (cols + 1) + bx + 1] = cnt;
}

// The summed-area table of one level from the block counts k_cur_mask stored: one CTA per image.
__global__ void __launch_bounds__(256)
k_cur_sat(int* __restrict__ sat, size_t sat_per_image, size_t sat_off, int w, int h) {
  int* S = sat + blockIdx.x * sat_per_image + sat_off;
  const int W = sat_cols(w), H = sat_rows(h);
  for (int i = threadIdx.x; i < W; i += blockDim.x) S[i] = 0;
  for (int j = threadIdx.x; j < H; j += blockDim.x) S[(size_t)j * W] = 0;
  __syncthreads();
  for (int j = 1 + threadIdx.x; j < H; j += blockDim.x) {   // rows
    int acc = 0;
    for (int i = 1; i < W; ++i) { acc += S[(size_t)j * W + i]; S[(size_t)j * W + i] = acc; }
  }
  __syncthreads();
  for (int i = 1 + threadIdx.x; i < W; i += blockDim.x) {   // columns
    int acc = 0;
    for (int j = 1; j < H; ++j) { acc += S[(size_t)j * W + i]; S[(size_t)j * W + i] = acc; }
  }
}

// {S, last selected linear index} of one (image, level) from its selection mask: one warp each
__global__ void k_sel_info(const uint32_t* __restrict__ masks, size_t mask_words_per_image, size_t mask_off, int words,
                           int* __restrict__ sel_info, int sel_info_per_image, int level) {
  const int img = blockIdx.x, lane = threadIdx.x;
  const uint32_t* m = masks + img * mask_words_per_image + mask_off;
  int cnt = 0, last = -1;
  for (int i = lane; i < words; i += 32) {
    const uint32_t v = m[i];
    cnt += __popc(v);
    if (v) last = i * 32 + 31 - __clz(v);     // i increases: the lane's last non-empty word wins
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    cnt += __shfl_xor_sync(0xffffffffu, cnt, off);
    last = max(last, __shfl_xor_sync(0xffffffffu, last, off));
  }
  if (lane == 0) {
    sel_info[img * sel_info_per_image + 2 * level] = cnt;
    sel_info[img * sel_info_per_image + 2 * level + 1] = last;
  }
}

// computeResidualsSse walks the point list two at a time and skips the last point of an odd list
// (dense_tracking_impl.cpp:169): that point is unselected in the reference plane.  Runs after k_sel_info.
__global__ void k_drop_odd_last(float2* __restrict__ planes, size_t planes_per_image, size_t rec_off, int nbands, int w,
                                const int* __restrict__ sel_info, int sel_info_per_image, int level, int nimg) {
  const int img = blockIdx.x * blockDim.x + threadIdx.x;
  if (img >= nimg) return;
  const int S = sel_info[img * sel_info_per_image + 2 * level], last = sel_info[img * sel_info_per_image + 2 * level + 1];
  if ((S & 1) && last >= 0) {
    const int y = last / w, x = last - y * w;
    float2* rec = planes + img * planes_per_image + rec_off;
    rec[rec_cell(x, y, nbands)].y = __int_as_float(0x7fc00000);
  }
}

// recompute the selection mask and the reference plane of one level for non-default thresholds (kMasked: usable = the
// level's usable bits, which the selection keeps honouring)
template <bool kMasked>
__global__ void k_reselect(const float2* __restrict__ P0, float2* __restrict__ rec, int nbands, int w, int h, int pitch,
                           uint32_t* __restrict__ mask, float ti, float td, const uint32_t* __restrict__ usable) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int n = w * h;
  bool sel = false;
  if (idx < n) {
    const int y = idx / w, x = idx - y * w;
    const size_t plane = (size_t)pitch * h, o = (size_t)y * pitch + x;
    const float2* P2 = P0 + plane;
    const size_t rc = rec_cell(x, y, nbands);
    const int xp = max(x - 1, 0), xn = min(x + 1, w - 1), yp = max(y - 1, 0), yn = min(y + 1, h - 1);
    const float2 a = P0[o], b = rec[rc + kRecP1];
    const float zx = (P2[(size_t)y * pitch + xn].y - P2[(size_t)y * pitch + xp].y) * 0.5f;
    const float zy = (P2[(size_t)yn * pitch + x].y - P2[(size_t)yp * pitch + x].y) * 0.5f;
    sel = !is_nan(a.y) && (fabsf(b.x) > ti || fabsf(b.y) > ti || fabsf(zx) > td || fabsf(zy) > td);
    if (kMasked) sel = sel && bit_set(usable, idx);
    rec[rc] = make_float2(a.x, sel ? a.y : __int_as_float(0x7fc00000));
  }
  unsigned m = __ballot_sync(0xffffffffu, sel);
  if ((threadIdx.x & 31) == 0 && idx < ((n + 31) / 32) * 32) mask[idx >> 5] = m;
}

// point-cloud template tx[x] = (x - ox)/fx, ty[y] = (y - oy)/fy (IEEE division, rgbd_image.cpp:197-198)
__global__ void k_template(float* __restrict__ tmpl, size_t tmpl_per_image, size_t off, int w, int h, float fx,
                           float fy, float ox, float oy) {
  int img = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  float* t = tmpl + img * tmpl_per_image + off;
  if (i < w) t[i] = __fdiv_rn((float)i - ox, fx);
  else if (i < w + h) t[i] = __fdiv_rn((float)(i - w) - oy, fy);
}

// The rectifying remap (dvo_b200_pyramid_create_rectified_batch): one thread per output pixel of one image.  Bilinear
// intensity in a fixed order with every operation rounded to nearest (no contraction), the nearest tap's depth, NaN / NaN
// where the map points outside [0, in_w-1] x [0, in_h-1].  kMasked: the pixel is usable iff it is valid and its four taps
// are.  The outputs are packed planes of w*h elements per image, the layout of a staged FLOAT32 upload.  kZbuf (a
// registered create): Z is not read; dZ holds k_register_scatter's z-buffer, whose untouched pixels become NaN, valid
// map or not.
template <bool kRaw, bool kMasked, bool kZbuf = false>
__global__ void __launch_bounds__(256)
k_rectify(SrcPlane I, SrcPlane Z, float zscale, SrcPlane M, const float* __restrict__ map_x, const float* __restrict__ map_y,
          int in_w, int in_h, int n, float* __restrict__ dI, float* __restrict__ dZ, uint8_t* __restrict__ dM) {
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float sx = __ldg(map_x + i), sy = __ldg(map_y + i);
  const float nanv = __int_as_float(0x7fc00000);
  float v = nanv, z = nanv;
  bool usable = false;
  if (sx >= 0.f && sx <= (float)(in_w - 1) && sy >= 0.f && sy <= (float)(in_h - 1)) {
    const int x0 = min((int)floorf(sx), in_w - 2), y0 = min((int)floorf(sy), in_h - 2);
    const float ax = __fsub_rn(sx, (float)x0), ay = __fsub_rn(sy, (float)y0);
    const float bx = __fsub_rn(1.f, ax), by = __fsub_rn(1.f, ay);
    const size_t o = I.at(img, y0, x0);
    const float i00 = load_intensity<kRaw>(I.data, o), i10 = load_intensity<kRaw>(I.data, o + 1);
    const float i01 = load_intensity<kRaw>(I.data, o + I.pitch), i11 = load_intensity<kRaw>(I.data, o + I.pitch + 1);
    const float top = __fadd_rn(__fmul_rn(bx, i00), __fmul_rn(ax, i10));
    const float bot = __fadd_rn(__fmul_rn(bx, i01), __fmul_rn(ax, i11));
    v = __fadd_rn(__fmul_rn(by, top), __fmul_rn(ay, bot));
    if (!kZbuf) z = load_depth<kRaw>(Z.data, Z.at(img, y0 + (ay >= 0.5f), x0 + (ax >= 0.5f)), zscale);
    if (kMasked) {
      const uint8_t* m = reinterpret_cast<const uint8_t*>(M.data) + M.at(img, y0, x0);
      usable = __ldg(m) && __ldg(m + 1) && __ldg(m + M.pitch) && __ldg(m + M.pitch + 1);
    }
  }
  const size_t out = (size_t)img * n + i;
  if (kZbuf) {
    const float zb = dZ[out];
    z = __float_as_uint(zb) == 0xffffffffu ? nanv : zb;
  }
  dI[out] = v;
  dZ[out] = z;
  if (kMasked) dM[out] = usable ? 1 : 0;
}

// Depth registration (dvo_b200_pyramid_create_registered_batch): the geometry of a dvo_b200_depth_registration, by value.
struct RegGeometry {
  int dw, dh, w, h;
  float R[9], t[3], K[4];
};

// ((r0*X + r1*Y) + r2*Z) + t, every operation rounded to nearest
__device__ __forceinline__ float reg_row(float r0, float r1, float r2, float t, float X, float Y, float Z) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(r0, X), __fmul_rn(r1, Y)), __fmul_rn(r2, Z)), t);
}

// The forward projection of the header, one thread per depth pixel of one image: Zc of the pixel's centre ray goes into
// every colour pixel of the footprint of its four corner rays through atomicMin on the float's bits, which order as
// unsigned ints for positive floats.  zbuf: packed w*h words per image, 0xffffffff where nothing has landed.  The result is
// the minimum over the covering pixels, whatever order the threads run in.
template <bool kRaw>
__global__ void __launch_bounds__(256)
k_register_scatter(SrcPlane Z, float zscale, RegGeometry g, const float* __restrict__ rays, unsigned* __restrict__ zbuf) {
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int npx = g.dw * g.dh;
  if (i >= npx) return;
  const int v = i / g.dw, u = i - v * g.dw;
  const float d = load_depth<kRaw>(Z.data, Z.at(img, v, u), zscale);
  if (!(d > 0.f) || !isfinite(d)) return;
  const float zc = reg_row(g.R[6], g.R[7], g.R[8], g.t[2], __fmul_rn(__ldg(rays + i), d), __fmul_rn(__ldg(rays + npx + i), d), d);
  if (!(zc > 0.f)) return;
  const float* kx = rays + 2 * (size_t)npx;
  const float* ky = kx + (size_t)(g.dw + 1) * (g.dh + 1);
  float xmin = INFINITY, xmax = -INFINITY, ymin = INFINITY, ymax = -INFINITY;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const size_t k = (size_t)(v + (c >> 1)) * (g.dw + 1) + u + (c & 1);
    const float X = __fmul_rn(__ldg(kx + k), d), Y = __fmul_rn(__ldg(ky + k), d);
    const float zk = reg_row(g.R[6], g.R[7], g.R[8], g.t[2], X, Y, d);
    if (!(zk > 0.f)) return;
    const float x = __fadd_rn(__fmul_rn(g.K[0], __fdiv_rn(reg_row(g.R[0], g.R[1], g.R[2], g.t[0], X, Y, d), zk)), g.K[2]);
    const float y = __fadd_rn(__fmul_rn(g.K[1], __fdiv_rn(reg_row(g.R[3], g.R[4], g.R[5], g.t[1], X, Y, d), zk)), g.K[3]);
    if (!(fabsf(x) < 1048576.f) || !(fabsf(y) < 1048576.f)) return;
    xmin = fminf(xmin, x); xmax = fmaxf(xmax, x);
    ymin = fminf(ymin, y); ymax = fmaxf(ymax, y);
  }
  const int x0 = (int)ceilf(xmin), x1 = (int)ceilf(xmax), y0 = (int)ceilf(ymin), y1 = (int)ceilf(ymax);
  if (x1 - x0 > DVO_B200_REGISTRATION_MAX_FOOTPRINT || y1 - y0 > DVO_B200_REGISTRATION_MAX_FOOTPRINT) return;
  const int xa = max(x0, 0), xb = min(x1, g.w), ya = max(y0, 0), yb = min(y1, g.h);
  unsigned* zb = zbuf + (size_t)img * g.w * g.h;
  const unsigned bits = __float_as_uint(zc);
  for (int y = ya; y < yb; ++y)
    for (int x = xa; x < xb; ++x) atomicMin(zb + (size_t)y * g.w + x, bits);
}

// The registered create's finish without a rectifier, one thread per colour pixel of one image: the packed float32
// intensity of the colour frame (as given, or 8-bit grey converted exactly), and NaN depth where the z-buffer is untouched.
template <bool kRaw>
__global__ void __launch_bounds__(256)
k_register_finish(SrcPlane I, int w, int n, float* __restrict__ dI, float* __restrict__ dZ) {
  const int img = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int y = i / w, x = i - y * w;
  const size_t out = (size_t)img * n + i;
  dI[out] = load_intensity<kRaw>(I.data, I.at(img, y, x));
  if (__float_as_uint(dZ[out]) == 0xffffffffu) dZ[out] = __int_as_float(0x7fc00000);
}

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

template <bool kLevel0, bool kRaw, typename... Args>
void launch_finish(bool masked, dim3 g, cudaStream_t st, Args... a) {
  if (masked) k_pyr_finish<kLevel0, kRaw, true><<<g, 256, 0, st>>>(a...);
  else k_pyr_finish<kLevel0, kRaw, false><<<g, 256, 0, st>>>(a...);
}

}  // namespace

int ensure_stage(dvo_b200_ctx* ctx, size_t dev_bytes, size_t host_bytes) {
  if (dev_bytes > ctx->d_stage_bytes) {
    if (ctx->d_stage) { cudaStreamSynchronize(ctx->stream); cudaFree(ctx->d_stage); ctx->d_stage = nullptr; ctx->d_stage_bytes = 0; }
    DVO_CUDA(ctx, cudaMalloc(&ctx->d_stage, dev_bytes));
    ctx->d_stage_bytes = dev_bytes;
  }
  if (host_bytes > ctx->h_stage_bytes) {
    if (ctx->h_stage) { cudaStreamSynchronize(ctx->stream); cudaFreeHost(ctx->h_stage); ctx->h_stage = nullptr; ctx->h_stage_bytes = 0; }
    DVO_CUDA(ctx, cudaMallocHost(&ctx->h_stage, host_bytes));
    ctx->h_stage_bytes = host_bytes;
  }
  return 0;
}

static void destroy_slab(Slab* s) {
  for (auto& u : s->foreign_uses) {   // another context's queued work may still read the slab
    cudaEventSynchronize(u.second);
    cudaEventDestroy(u.second);
  }
  cudaFree(s->base);
  if (s->ready) cudaEventDestroy(s->ready);
  delete s;
}

static Slab* acquire_slab(dvo_b200_ctx* ctx, size_t bytes) {
  SlabPool& pool = *ctx->pool;
  std::lock_guard<std::mutex> lock(pool.mu);   // pyramids may be released by another host thread (see pyramid_free)
  auto it = pool.free.find(bytes);
  if (it != pool.free.end()) {
    Slab* s = it->second;
    pool.free.erase(it);
    s->refs = 0;
    // the build that follows rewrites the slab on this stream: after every other context's work that read it
    for (auto& u : s->foreign_uses) cudaStreamWaitEvent(ctx->stream, u.second, 0);
    return s;
  }
  void* p = nullptr;
  if (cudaMalloc(&p, bytes) != cudaSuccess) {
    // drop the pool and retry once
    for (auto& kv : pool.free) destroy_slab(kv.second);
    pool.free.clear();
    cudaGetLastError();
    if (cudaMalloc(&p, bytes) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  }
  Slab* s = new Slab;
  s->base = p; s->bytes = bytes; s->refs = 0; s->pool = ctx->pool;
  return s;
}

// Called from any host thread, possibly after the owning context has been destroyed.
void pyramid_free(dvo_b200_pyramid* p) {
  Slab* s = p->slab;
  delete p;
  if (!s) return;
  std::shared_ptr<SlabPool> pool = s->pool;    // keeps the pool alive while its mutex is held
  std::lock_guard<std::mutex> lock(pool->mu);
  if (--s->refs == 0) {
    if (pool->closed) { DeviceScope dev(pool->device); destroy_slab(s); }
    else pool->free.insert({s->bytes, s});
  }
}

void wait_for_pyramid(dvo_b200_ctx* ctx, const dvo_b200_pyramid* p) {
  // Also for the context's own pyramids: the event may have been re-recorded by another context's re-selection, and
  // waiting on an event last recorded on this very stream costs nothing.
  if (p->slab && p->slab->ready) cudaStreamWaitEvent(ctx->stream, p->slab->ready, 0);
}

int note_foreign_use(dvo_b200_ctx* ctx, const dvo_b200_pyramid* p) {
  Slab* s = p->slab;
  if (!s || s->pool == ctx->pool) return 0;   // the owner's own work is ordered before its later builds by its stream
  std::lock_guard<std::mutex> lock(s->pool->mu);
  cudaEvent_t e = nullptr;
  for (auto& u : s->foreign_uses)
    if (u.first == ctx->uid) e = u.second;
  if (!e) {
    DVO_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    s->foreign_uses.push_back({ctx->uid, e});
  }
  DVO_CUDA(ctx, cudaEventRecord(e, ctx->stream));
  return 0;
}

// The context goes away: free what is pooled, and have slabs still referenced by live pyramids freed on release.
void pool_close(dvo_b200_ctx* ctx) {
  if (!ctx->pool) return;
  std::lock_guard<std::mutex> lock(ctx->pool->mu);
  for (auto& kv : ctx->pool->free) destroy_slab(kv.second);
  ctx->pool->free.clear();
  ctx->pool->closed = true;
}

int remap_batch(dvo_b200_ctx* ctx, const dvo_b200_rectifier* rect, const dvo_b200_depth_registration* reg, int n, SrcPlane I,
                SrcPlane Z, int raw, float zscale, SrcPlane M, float* dI, float* dZ, uint8_t* dM) {
  ProfScope prof(ctx, 3, reg ? 2 : 1);
  const int npx = reg ? reg->w * reg->h : rect->w * rect->h;
  const dim3 gc((npx + 255) / 256, n);
  cudaStream_t st = ctx->stream;
  if (reg) {
    DVO_CUDA(ctx, cudaMemsetAsync(dZ, 0xff, (size_t)npx * n * sizeof(float), st));   // the empty z-buffer
    RegGeometry geo;
    geo.dw = reg->dw; geo.dh = reg->dh; geo.w = reg->w; geo.h = reg->h;
    for (int k = 0; k < 9; ++k) geo.R[k] = reg->R[k];
    for (int k = 0; k < 3; ++k) geo.t[k] = reg->t[k];
    for (int k = 0; k < 4; ++k) geo.K[k] = reg->K[k];
    const dim3 gs((reg->dw * reg->dh + 255) / 256, n);
    unsigned* zbuf = reinterpret_cast<unsigned*>(dZ);
    if (raw) k_register_scatter<true><<<gs, 256, 0, st>>>(Z, zscale, geo, reg->rays, zbuf);
    else k_register_scatter<false><<<gs, 256, 0, st>>>(Z, zscale, geo, reg->rays, zbuf);
  }
  if (rect) {   // intensity and masks through the map; depth from the map's nearest tap, or from the z-buffer
    using Rectify = void (*)(SrcPlane, SrcPlane, float, SrcPlane, const float*, const float*, int, int, int, float*, float*, uint8_t*);
    static const Rectify kernels[2][2][2] = {   // [raw][masked][z-buffer]
        {{k_rectify<false, false, false>, k_rectify<false, false, true>}, {k_rectify<false, true, false>, k_rectify<false, true, true>}},
        {{k_rectify<true, false, false>, k_rectify<true, false, true>}, {k_rectify<true, true, false>, k_rectify<true, true, true>}}};
    kernels[raw ? 1 : 0][M.data ? 1 : 0][reg ? 1 : 0]<<<gc, 256, 0, st>>>(I, Z, reg ? 0.f : zscale, M, rect->map, rect->map + npx,
                                                                          rect->in_w, rect->in_h, npx, dI, dZ, dM);
  } else if (raw) {
    k_register_finish<true><<<gc, 256, 0, st>>>(I, reg->w, npx, dI, dZ);
  } else {
    k_register_finish<false><<<gc, 256, 0, st>>>(I, reg->w, npx, dI, dZ);
  }
  ctx->launches += reg ? 2 : 1;
  return 0;
}

// I / Z: raw == 0: float32 intensity / float32 depth; raw == 1: 8-bit grey / 16-bit raw depth (depth = raw * zscale, 0 -> NaN)
// M: reference masks of bytes (nonzero = usable), or M.data == NULL.  Without masks the slab holds no usable bits and the
// build runs exactly the kernels it ran before masks existed.  mask_roles with DVO_B200_MASK_ROLE_CURRENT: the masks also
// act in the current role (k_cur_mask, k_cur_sat after the other kernels of each level); otherwise the build is the
// reference-mask build, kernel for kernel.  The planes are read where they lie, with their pitch and stride: staged
// uploads and the caller's device memory take the same kernels.
int pyramid_build_batch_input(dvo_b200_ctx* ctx, int n, SrcPlane I, SrcPlane Z, int raw, float zscale, int w, int h,
                              const float K[4], int levels, dvo_b200_pyramid** out, SrcPlane M, int mask_roles) {
  LevelInfo L[kMaxLevels];
  const std::string why = derive_levels(w, h, K, levels, L);   // the creates have refused a bad geometry already
  if (!why.empty()) return set_error(ctx, DVO_B200_ERR_INVALID_ARGUMENT, "pyramid: " + why);
  size_t plane_f2 = 0, mask_words = 0, tmpl_floats = 0, range_f2 = 0, sat_ints = 0;
  for (int l = 0; l < levels; ++l) {
    LevelInfo& q = L[l];
    q.plane_off = plane_f2; plane_f2 += 2 * (size_t)q.pitch * q.h;                       // P0, P2 (row-major, even pitch)
    q.rec_off = plane_f2; plane_f2 += (size_t)q.nbands * q.nstrips * kRecF2;               // reference tile records
    q.mask_off = mask_words; mask_words += q.words;
    q.tmpl_off = tmpl_floats; tmpl_floats += (size_t)((q.w + q.h + 3) & ~3);   // every level's tx[] starts 16-byte aligned (bulk copies)
    q.range_off = range_f2; range_f2 += (size_t)q.nbands * q.nstrips;
    q.sat_off = sat_ints; sat_ints += (size_t)sat_cols(q.w) * sat_rows(q.h);
  }
  plane_f2 = align_up(plane_f2, 32);          // keep every image 256-byte aligned
  mask_words = align_up(mask_words, 64);
  tmpl_floats = align_up(tmpl_floats + kTileW, 64);   // lanes past a partial band read (and discard) up to kTileW floats beyond tx[w]
  range_f2 = align_up(range_f2, 32);
  sat_ints = align_up(sat_ints, 64);
  const int sel_ints = 2 * kMaxLevels;
  size_t bytes_planes = (size_t)n * plane_f2 * sizeof(float2);
  size_t bytes_masks = (size_t)n * mask_words * sizeof(uint32_t);
  size_t bytes_tmpl = (size_t)n * tmpl_floats * sizeof(float);
  size_t bytes_sel = align_up((size_t)n * sel_ints * sizeof(int), 256);
  size_t bytes_range = (size_t)n * range_f2 * sizeof(float2);
  const bool masked = M.data != nullptr;
  size_t bytes_usable = masked ? bytes_masks : 0;   // usable bits: the layout of the selection masks
  const bool cur_masked = masked && (mask_roles & DVO_B200_MASK_ROLE_CURRENT) != 0;
  size_t bytes_sat = cur_masked ? (size_t)n * sat_ints * sizeof(int) : 0;   // unusable-pixel summaries, after the usable bits
  size_t total = bytes_planes + bytes_masks + bytes_tmpl + bytes_sel + bytes_range + bytes_usable + bytes_sat;
  Slab* slab = acquire_slab(ctx, total);
  if (!slab) return set_error(ctx, DVO_B200_ERR_OUT_OF_MEMORY, "pyramid: cudaMalloc failed");
  char* base = (char*)slab->base;
  float2* planes = (float2*)base;
  uint32_t* masks = (uint32_t*)(base + bytes_planes);
  float* tmpl = (float*)(base + bytes_planes + bytes_masks);
  int* sel = (int*)(base + bytes_planes + bytes_masks + bytes_tmpl);
  float2* ranges = (float2*)(base + bytes_planes + bytes_masks + bytes_tmpl + bytes_sel);
  uint32_t* usable = masked ? (uint32_t*)(base + bytes_planes + bytes_masks + bytes_tmpl + bytes_sel + bytes_range) : nullptr;
  int* sat = cur_masked ? (int*)(base + bytes_planes + bytes_masks + bytes_tmpl + bytes_sel + bytes_range + bytes_usable) : nullptr;

  cudaStream_t st = ctx->stream;
  {
    ProfScope prof(ctx, 3, (cur_masked ? 9 : masked ? 7 : 6) * levels - 1);
    const int T = 256;
    // the 2x2 blocks of level 0 start at two-element boundaries: base address, row pitch and image stride even (in elements)
    const size_t two_elems = raw ? 2 : 2 * sizeof(float);
    const int aligned = (uintptr_t)I.data % two_elems == 0 && I.pitch % 2 == 0 && I.stride % 2 == 0 ? 1 : 0;
    const SrcPlane none{nullptr, 0, 0};
    for (int l = 0; l < levels; ++l) {
      const LevelInfo& q = L[l];
      dim3 gt((q.w + q.h + T - 1) / T, n);
      k_template<<<gt, T, 0, st>>>(tmpl, tmpl_floats, q.tmpl_off, q.w, q.h, q.fx, q.fy, q.ox, q.oy);
      ctx->launches += 1;
      if (l == 0) continue;   // level 0 takes its intensity from the input image
      dim3 g((q.n + T - 1) / T, n);
      if (l == 1 && raw) k_pyr_intensity_down<true, true><<<g, T, 0, st>>>(I, aligned, planes, plane_f2, 0, L[0].pitch, q.plane_off, q.w, q.h, q.pitch);
      else if (l == 1) k_pyr_intensity_down<true, false><<<g, T, 0, st>>>(I, aligned, planes, plane_f2, 0, L[0].pitch, q.plane_off, q.w, q.h, q.pitch);
      else k_pyr_intensity_down<false, false><<<g, T, 0, st>>>(none, 0, planes, plane_f2, L[l - 1].plane_off, L[l - 1].pitch, q.plane_off, q.w, q.h, q.pitch);
      ctx->launches += 1;
    }
    for (int l = 0; l < levels; ++l) {
      const LevelInfo& q = L[l];
      dim3 g((q.words * 32 + T - 1) / T, n);
      if (masked) {
        if (l == 0) k_usable<true><<<g, T, 0, st>>>(M, usable, mask_words, 0, 0, q.mask_off, q.w, q.h);
        else k_usable<false><<<g, T, 0, st>>>(none, usable, mask_words, L[l - 1].mask_off, L[l - 1].w, q.mask_off, q.w, q.h);
        ctx->launches += 1;
      }
      if (l == 0 && raw) launch_finish<true, true>(masked, g, st, I, Z, zscale, planes, plane_f2, q.plane_off, q.rec_off, q.nbands, q.w, q.h, q.pitch, l, masks, mask_words, q.mask_off, 0.f, 0.f, usable);
      else if (l == 0) launch_finish<true, false>(masked, g, st, I, Z, zscale, planes, plane_f2, q.plane_off, q.rec_off, q.nbands, q.w, q.h, q.pitch, l, masks, mask_words, q.mask_off, 0.f, 0.f, usable);
      else if (raw) launch_finish<false, true>(masked, g, st, I, Z, zscale, planes, plane_f2, q.plane_off, q.rec_off, q.nbands, q.w, q.h, q.pitch, l, masks, mask_words, q.mask_off, 0.f, 0.f, usable);
      else launch_finish<false, false>(masked, g, st, I, Z, zscale, planes, plane_f2, q.plane_off, q.rec_off, q.nbands, q.w, q.h, q.pitch, l, masks, mask_words, q.mask_off, 0.f, 0.f, usable);
      k_sel_info<<<n, 32, 0, st>>>(masks, mask_words, q.mask_off, q.words, sel, sel_ints, l);
      k_drop_odd_last<<<(n + 127) / 128, 128, 0, st>>>(planes, plane_f2, q.rec_off, q.nbands, q.w, sel, sel_ints, l, n);
      const int ntiles = q.nbands * q.nstrips;
      k_rec_fill<<<dim3((ntiles * kTileW + T - 1) / T, n), T, 0, st>>>(planes, plane_f2, q.rec_off, q.nbands, ntiles, q.w, q.h,
                                                                              tmpl, tmpl_floats, q.tmpl_off);
      ctx->launches += 1;
      const dim3 gr((ntiles + 7) / 8, n);
      if (masked)
        k_tile_range<true><<<gr, 256, 0, st>>>(planes, plane_f2, q.plane_off, q.w, q.h, q.pitch, q.nbands, ntiles, ranges, range_f2,
                                               q.range_off, usable, mask_words, q.mask_off);
      else
        k_tile_range<false><<<gr, 256, 0, st>>>(planes, plane_f2, q.plane_off, q.w, q.h, q.pitch, q.nbands, ntiles, ranges, range_f2,
                                                q.range_off, nullptr, 0, 0);
      ctx->launches += 4;
      if (cur_masked) {
        const int nblk = (sat_cols(q.w) - 1) * (sat_rows(q.h) - 1);
        k_cur_mask<<<dim3((nblk + T - 1) / T, n), T, 0, st>>>(planes, plane_f2, q.plane_off, q.w, q.h, q.pitch, usable, mask_words,
                                                                q.mask_off, sat, sat_ints, q.sat_off);
        k_cur_sat<<<n, T, 0, st>>>(sat, sat_ints, q.sat_off, q.w, q.h);
        ctx->launches += 2;
      }
    }
  }
  DVO_CUDA(ctx, cudaGetLastError());
  if (!slab->ready) DVO_CUDA(ctx, cudaEventCreateWithFlags(&slab->ready, cudaEventDisableTiming));
  DVO_CUDA(ctx, cudaEventRecord(slab->ready, st));
  for (int i = 0; i < n; ++i) {
    dvo_b200_pyramid* p = new dvo_b200_pyramid;
    p->ctx = ctx; p->device = ctx->device; p->refcount.store(1); p->levels = levels;
    std::memcpy(p->L, L, sizeof(LevelInfo) * levels);
    p->slab = slab; slab->refs++;
    p->planes = planes + (size_t)i * plane_f2;
    p->sel_mask = masks + (size_t)i * mask_words;
    p->sel_info = sel + (size_t)i * sel_ints;
    p->tmpl = tmpl + (size_t)i * tmpl_floats;
    p->tile_range = ranges + (size_t)i * range_f2;
    p->usable = masked ? usable + (size_t)i * mask_words : nullptr;
    p->cur_sat = cur_masked ? sat + (size_t)i * sat_ints : nullptr;
    p->mask_roles = !masked ? 0 : cur_masked ? (DVO_B200_MASK_ROLE_REFERENCE | DVO_B200_MASK_ROLE_CURRENT) : DVO_B200_MASK_ROLE_REFERENCE;
    p->id = ctx->next_pyramid_id++;
    out[i] = p;
  }
  return 0;
}

// The selection (mask, {S, last}, the Zsel channel of the reference tile records) is state of the PYRAMID, shared by every context that aligns
// against it, while the reference keeps it per tracker (PointSelection, point_selection.cpp:100-113).  Contexts that use
// the same thresholds -- every caller in dvo_slam: one configuration per tracker family -- never get here twice.  A context
// that asks for other thresholds rewrites the selection on its stream; the host-side state is guarded by sel_mu and the
// slab's ready event is re-recorded, so a context that enqueues work on this pyramid LATER waits for the rewrite.  What is
// not supported: two contexts aligning against one reference pyramid with different thresholds at the same time
// (INTEGRATION.md, limits).
int pyramid_reselect(dvo_b200_ctx* ctx, dvo_b200_pyramid* p, float ti, float td) {
  std::lock_guard<std::mutex> lock(p->sel_mu);
  if (p->sel_ti == ti && p->sel_td == td) return 0;
  cudaStream_t st = ctx->stream;
  ProfScope prof(ctx, 4, 3 * p->levels);
  for (int l = 0; l < p->levels; ++l) {
    const LevelInfo& q = p->L[l];
    const int T = 256;
    const int blocks = (q.words * 32 + T - 1) / T;
    if (p->usable)
      k_reselect<true><<<blocks, T, 0, st>>>(p->planes + q.plane_off, p->planes + q.rec_off, q.nbands, q.w, q.h, q.pitch,
                                             p->sel_mask + q.mask_off, ti, td, p->usable + q.mask_off);
    else
      k_reselect<false><<<blocks, T, 0, st>>>(p->planes + q.plane_off, p->planes + q.rec_off, q.nbands, q.w, q.h, q.pitch,
                                              p->sel_mask + q.mask_off, ti, td, nullptr);
    k_sel_info<<<1, 32, 0, st>>>(p->sel_mask, 0, q.mask_off, q.words, p->sel_info, 0, l);
    k_drop_odd_last<<<1, 32, 0, st>>>(p->planes, 0, q.rec_off, q.nbands, q.w, p->sel_info, 0, l, 1);
    ctx->launches += 3;
  }
  DVO_CUDA(ctx, cudaGetLastError());
  if (p->slab && p->slab->ready) DVO_CUDA(ctx, cudaEventRecord(p->slab->ready, st));
  p->sel_ti = ti; p->sel_td = td;
  return 0;
}

}  // namespace dvo_b200
