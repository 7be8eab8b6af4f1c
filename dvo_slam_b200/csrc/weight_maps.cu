// weight_maps.cu -- the weight maps of dvo_b200_match_batch_maps (include/dvo_b200.h, "weight maps"): after the level kernels
// of a match, one kernel reads each pair's final state and writes its Student-t weights, residuals and outlier mask at the
// kept iteration's pose.  The level kernels are not touched: the residual of a pixel is recomputed from the pyramids with
// the level kernel's own pixel functions (stages.cuh), whose operations decide the bits.
#include "common.cuh"
#define DVO_B200_STAGES_NO_DUMP   // the record dump belongs to tracker.cu (stages.cuh)
#include "stages.cuh"

#include <algorithm>

namespace dvo_b200 {

namespace {

constexpr int kMapsBlockX = 32, kMapsBlockY = 8;

// One launch of k_weight_maps: the batch's level-L geometry (the pyramids of a batch share their sizes) and the outputs, with
// dvo_b200_weight_maps's layout (NULL: not written).
struct MapsLaunch {
  float* plane[3];              // weight, residual_i, residual_z
  int64_t row_bytes[3], image_bytes[3];
  uint8_t* mask;
  int64_t mask_row_bytes, mask_image_bytes;
  float mask_weight;
  double* estimate;             // 16 per pair
  float* precision;             // 4 per pair
  int w, h, pitch, nbands;      // level L
  int w0, h0, level;            // level 0, and L
  int corrected;                // DVO_B200_ESTIMATOR_CORRECTED: the odd last selected point is a constraint
};

// What every pixel of a pair needs, computed once per block by thread 0 (the fp64 se3 matrix of T^ and the K T chain would
// otherwise be recomputed by each of the ~157 M threads of a 512-pair step).
struct PairConsts {
  float kt[12];         // K_cur,L * float(T^)[0:3, :]
  float P[4];           // P^
  float alpha, beta;    // the photometric mode's (alpha, beta), as float
  int ok;               // the Result is defined (k_finalize's `ok`)
  int odd_y, odd_x;     // the corrected estimator's odd last point (odd_y = -1: none)
  float odd_z;
};

// One thread per level-L pixel (x, y) of pair blockIdx.z: the residual record of stage A at the kept iteration's K T (the
// reference's (I, Zsel) from its tile record, the template, four taps of the current P0 -- Z' is NaN at the current role's
// unusable pixels, so the blend's NaN test rejects them as the level kernel does), the Student-t weight at P^, and the
// mask bytes of the pixel's 2^L x 2^L level-0 footprint in the same pass.  The grid covers ceil(w0 / 2^L) x ceil(h0 / 2^L)
// parents, so that the level-0 pixels past an odd size (no level-L parent) get their 1 from a thread too.
__global__ void __launch_bounds__(kMapsBlockX * kMapsBlockY)
k_weight_maps(const PairState* __restrict__ states, const AffineState* __restrict__ affine, const PairLevel* __restrict__ pls,
              const MapsLaunch m) {
  __shared__ PairConsts pc;
  const int pair = blockIdx.z;
  const int x = blockIdx.x * kMapsBlockX + threadIdx.x, y = blockIdx.y * kMapsBlockY + threadIdx.y;
  const PairLevel& pl = pls[pair];
  const float nanv = __int_as_float(0x7fc00000);
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    const PairState& st = states[pair];
    const bool ok = st.result_defined();
    // P^: after a rejected last iteration (LogLikelihoodDecreased) pair_mid_warp has moved the kept iteration's precision to
    // precision_prev; after an accepted one it is still `precision`
    const float* Pk = st.termination == DVO_B200_TERM_LOG_LIKELIHOOD_DECREASED ? st.precision_prev : st.precision;
    double T[16];
    se3_matrix(st.estimate, T);
    kt_of(T, pl, pc.kt);   // K T from T^: PairState::kt may belong to a rejected iteration
    for (int i = 0; i < 4; ++i) pc.P[i] = Pk[i];
    pc.alpha = affine ? (float)affine[pair].ab[0] : 1.f;
    pc.beta = affine ? (float)affine[pair].ab[1] : 0.f;
    pc.ok = ok;
    pc.odd_y = -1; pc.odd_x = 0; pc.odd_z = 0.f;
    if (m.corrected) {   // the odd last point is unselected in the tile records (k_drop_odd_last); the corrected estimator keeps it
      LevelGeom g;
      g.w = m.w; g.pitch = m.pitch;
      const OddPoint odd = load_odd_point(pl, g);
      pc.odd_y = odd.y; pc.odd_x = odd.x; pc.odd_z = odd.z;
    }
    if (blockIdx.x == 0 && blockIdx.y == 0) {
      if (m.estimate)
        for (int i = 0; i < 16; ++i) m.estimate[(size_t)pair * 16 + i] = T[i];
      if (m.precision)
        for (int i = 0; i < 4; ++i) m.precision[(size_t)pair * 4 + i] = ok ? Pk[i] : nanv;
    }
  }
  __syncthreads();
  const bool in_level = x < m.w && y < m.h;
  bool outlier = false;
  if (in_level) {
    float ei = nanv, ez = nanv, wgt = nanv;
    const float2 rec = __ldg(pl.r0 + rec_cell(x, y, m.nbands));   // (I, Zsel): Zsel NaN where the pixel is not a selected point
    const float z = (y == pc.odd_y && x == pc.odd_x) ? pc.odd_z : rec.y;
    if (pc.ok && z == z) {
      StageConsts c;
      c.k0 = pk(pc.kt[0], pc.kt[4]); c.k1 = pk(pc.kt[1], pc.kt[5]); c.k2 = pk(pc.kt[2], pc.kt[6]); c.k3 = pk(pc.kt[3], pc.kt[7]);
      c.k8 = pc.kt[8]; c.k9 = pc.kt[9]; c.k10 = pc.kt[10]; c.k11 = pc.kt[11];
      c.Pa = pk(pc.P[0], pc.P[1]); c.Pb = pk(pc.P[2], pc.P[3]);
      c.c_i = 1.0f / 255.0f;
      c.ubx = (float)(m.w - 2); c.uby = (float)(m.h - 2);
      c.first_iteration = 0;
      const float tx = __ldg(pl.rtmpl + x), ty = __ldg(pl.rtmpl + m.w + y);
      const PixelProjection p = project_pixel(tx, ty, z, c);
      const float Ir = affine ? ref_intensity<true>(rec.x, Brightness{pc.alpha, pc.beta}) : rec.x;
      // the four taps of stage A's residual_pixel, from the current P0 through L1 (a rejected point reads pixel (0, 0))
      const float2* t = pl.c0 + (size_t)p.v0 * m.pitch + p.u0;
      const f2 c00 = ldg_f2(t), c10 = ldg_f2(t + 1), c01 = ldg_f2(t + m.pitch), c11 = ldg_f2(t + m.pitch + 1);
      const float fu = lo(p.f), fv = hi(p.f), gu = lo(p.gq), gv = hi(p.gq);
      const f2 IZ = DVO_BLEND2(fu, fv, gu, gv, c00, c10, c01, c11);
      const float Zc = hi(IZ);
      const float e_z = __fsub_rn(Zc, p.Zt);
      const float e_i = __fmaf_rn(c.c_i, lo(IZ), __fmul_rn(-c.c_i, Ir));
      if (p.inb && Zc == Zc && e_z > __fmul_rn(-20.0f, depth_sigma(z))) {
        ei = e_i; ez = e_z;
        wgt = student_weight(c, false, ei, ez);
        outlier = wgt < m.mask_weight;
      }
    }
    const float v[3] = {wgt, ei, ez};
    for (int k = 0; k < 3; ++k)
      if (m.plane[k])
        *reinterpret_cast<float*>(reinterpret_cast<char*>(m.plane[k]) + pair * m.image_bytes[k] + y * m.row_bytes[k] + x * 4) = v[k];
  }
  if (m.mask) {
    const int s = 1 << m.level;
    const int x0 = x << m.level, y0 = y << m.level;
    if (x0 < m.w0 && y0 < m.h0) {
      uint8_t* base = m.mask + pair * m.mask_image_bytes;
      const int x1 = min(x0 + s, m.w0), y1 = min(y0 + s, m.h0);
      const uint8_t b = outlier ? 0 : 1;
      for (int yy = y0; yy < y1; ++yy)
        for (int xx = x0; xx < x1; ++xx) base[yy * m.mask_row_bytes + xx] = b;
    }
  }
}

// The outputs at `maps` (device memory) written in place: a plane's MapsLaunch entry is the caller's
void set_outputs(MapsLaunch& m, const dvo_b200_weight_maps& maps) {
  const dvo_b200_map_plane* pl[3] = {&maps.weight, &maps.residual_i, &maps.residual_z};
  for (int k = 0; k < 3; ++k) {
    m.plane[k] = static_cast<float*>(pl[k]->data);
    m.row_bytes[k] = pl[k]->row_bytes; m.image_bytes[k] = pl[k]->image_bytes;
  }
  m.mask = static_cast<uint8_t*>(maps.mask.data);
  m.mask_row_bytes = maps.mask.row_bytes; m.mask_image_bytes = maps.mask.image_bytes;
  m.estimate = maps.estimate; m.precision = maps.precision;
}

// DVO_B200_MAPS_HOST: the kernel writes packed maps into the device scratch ws.d_maps, at these offsets (weight, residual_i,
// residual_z, mask, estimate, precision); returns the bytes needed.
size_t host_scratch_layout(const dvo_b200_weight_maps& maps, int n, const dvo_b200_pyramid* ref0, int level, size_t off[6]) {
  const LevelInfo& L = ref0->L[level];
  const size_t map_bytes = sizeof(float) * (size_t)L.w * L.h, mask_bytes = (size_t)ref0->L[0].w * ref0->L[0].h;
  size_t at = 0;
  auto take = [&](bool used, size_t bytes) { const size_t o = at; if (used) at += (bytes * n + 255) / 256 * 256; return o; };
  off[0] = take(maps.weight.data != nullptr, map_bytes);
  off[1] = take(maps.residual_i.data != nullptr, map_bytes);
  off[2] = take(maps.residual_z.data != nullptr, map_bytes);
  off[3] = take(maps.mask.data != nullptr, mask_bytes);
  off[4] = take(maps.estimate != nullptr, 16 * sizeof(double));
  off[5] = take(maps.precision != nullptr, 4 * sizeof(float));
  return at;
}

}  // namespace

int weight_maps_prepare(dvo_b200_ctx* ctx, const dvo_b200_weight_maps& maps, int n, const dvo_b200_pyramid* ref0, int level) {
  if (maps.memory != DVO_B200_MAPS_HOST) return 0;
  size_t off[6];
  return grow(ctx, ctx->ws.d_maps, ctx->ws.cap_maps, host_scratch_layout(maps, n, ref0, level, off));
}

void weight_maps_launch(dvo_b200_ctx* ctx, const dvo_b200_weight_maps& maps, int n, const dvo_b200_pyramid* ref0, int level,
                        const PairState* d_states, const PairLevel* d_pls, const AffineState* d_affine) {
  Workspace& ws = ctx->ws;
  const LevelInfo& L = ref0->L[level];
  MapsLaunch m;
  m.mask_weight = maps.mask_weight;
  m.w = L.w; m.h = L.h; m.pitch = L.pitch; m.nbands = L.nbands;
  m.w0 = ref0->L[0].w; m.h0 = ref0->L[0].h; m.level = level;
  m.corrected = ctx->estimator == DVO_B200_ESTIMATOR_CORRECTED;
  set_outputs(m, maps);
  if (maps.memory == DVO_B200_MAPS_HOST) {   // packed, into the scratch weight_maps_prepare sized
    size_t off[6];
    host_scratch_layout(maps, n, ref0, level, off);
    char* s = ws.d_maps;
    const int64_t map_bytes = sizeof(float) * (int64_t)L.w * L.h;
    for (int k = 0; k < 3; ++k)
      if (m.plane[k]) { m.plane[k] = reinterpret_cast<float*>(s + off[k]); m.row_bytes[k] = sizeof(float) * L.w; m.image_bytes[k] = map_bytes; }
    if (m.mask) { m.mask = reinterpret_cast<uint8_t*>(s + off[3]); m.mask_row_bytes = m.w0; m.mask_image_bytes = (int64_t)m.w0 * m.h0; }
    if (m.estimate) m.estimate = reinterpret_cast<double*>(s + off[4]);
    if (m.precision) m.precision = reinterpret_cast<float*>(s + off[5]);
  }
  ProfScope prof(ctx, 2);
  const int sc = 1 << level;
  const int gx = std::max(L.w, (m.w0 + sc - 1) / sc), gy = std::max(L.h, (m.h0 + sc - 1) / sc);
  const dim3 grid((gx + kMapsBlockX - 1) / kMapsBlockX, (gy + kMapsBlockY - 1) / kMapsBlockY, n);
  k_weight_maps<<<grid, dim3(kMapsBlockX, kMapsBlockY), 0, ctx->stream>>>(d_states, d_affine, d_pls, m);
  ctx->launches++;
}

int weight_maps_copy_back(dvo_b200_ctx* ctx, const dvo_b200_weight_maps& maps, int n, const dvo_b200_pyramid* ref0, int level) {
  if (maps.memory != DVO_B200_MAPS_HOST) return 0;
  cudaStream_t st = ctx->stream;
  const char* s = ctx->ws.d_maps;
  const LevelInfo& L = ref0->L[level];
  size_t off[6];
  host_scratch_layout(maps, n, ref0, level, off);
  // into the caller's layout: one 2D copy of n * h rows where the caller's maps follow each other without a gap, else one per pair
  auto copy = [&](const dvo_b200_map_plane& dst, const char* src, size_t width, int h) -> int {
    if (!dst.data) return 0;
    if (dst.image_bytes == dst.row_bytes * h) {
      DVO_CUDA(ctx, cudaMemcpy2DAsync(dst.data, dst.row_bytes, src, width, width, (size_t)h * n, cudaMemcpyDeviceToHost, st));
    } else {
      for (int p = 0; p < n; ++p)
        DVO_CUDA(ctx, cudaMemcpy2DAsync(static_cast<char*>(dst.data) + p * dst.image_bytes, dst.row_bytes, src + p * width * h, width, width,
                                        (size_t)h, cudaMemcpyDeviceToHost, st));
    }
    ctx->d2h_bytes += (int64_t)(width * h * n);
    return 0;
  };
  const dvo_b200_map_plane* pl[3] = {&maps.weight, &maps.residual_i, &maps.residual_z};
  for (int k = 0; k < 3; ++k)
    if (int rc = copy(*pl[k], s + off[k], sizeof(float) * L.w, L.h)) return rc;
  if (int rc = copy(maps.mask, s + off[3], (size_t)ref0->L[0].w, ref0->L[0].h)) return rc;
  if (maps.estimate) {
    DVO_CUDA(ctx, cudaMemcpyAsync(maps.estimate, s + off[4], 16 * sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    ctx->d2h_bytes += 16 * sizeof(double) * n;
  }
  if (maps.precision) {
    DVO_CUDA(ctx, cudaMemcpyAsync(maps.precision, s + off[5], 4 * sizeof(float) * n, cudaMemcpyDeviceToHost, st));
    ctx->d2h_bytes += 4 * sizeof(float) * n;
  }
  return 0;
}

}  // namespace dvo_b200
